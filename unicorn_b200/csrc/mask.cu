// CondInst mask path (config 4): aligned-bilinear fusion of the mask branch, per-instance dynamic convolutions,
// RAFT-style convex upsampling, sigmoid, final aligned-bilinear upsample.
//   uc_aligned_bilinear_add   condinst/comm.py:5-27 + mask_branch.py:81-96 (x = x + aligned_bilinear(x_p, f))
//   uc_dynamic_masks          condinst/dynamic_mask_head.py:61-87 (parameter split), :172-225 (rel-coords + 3 grouped
//                             1x1 convs 10->8->8->1), :159-170 (convex upsample x up_rate), :284 (sigmoid);
//                             utils/boxes.py:138-145 (aligned_bilinear x d_rate of the scores)
// HBM-bound on the output (N x H x W fp32 masks); all arithmetic fp32.
#include "uc_common.h"
#include "../../include/unicorn_b200.h"
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>

namespace uc {

// aligned_bilinear(t, f)[i] samples the (replicate-padded) source at max(i - f/2, 0) / f with align_corners=True.
__device__ __forceinline__ void ab_coord(int i, int f, int n, int& i0, int& i1, float& frac) {
  const int ii = max(i - f / 2, 0);
  i0 = ii / f;
  frac = static_cast<float>(ii - i0 * f) / f;
  i1 = min(i0 + 1, n - 1);
  i0 = min(i0, n - 1);
}

// blockIdx.y = image: image b reads src + b * bs_src and updates dst + b * bs_dst
__global__ void __launch_bounds__(256) aligned_bilinear_add_kernel(const uint16_t* __restrict__ src, int lds, long bs_src, int hs, int ws,
                                                                    uint16_t* __restrict__ dst, int ldd, long bs_dst, int C, int f) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  src += blockIdx.y * bs_src;
  dst += blockIdx.y * bs_dst;
  const int C2 = C >> 1, hd = hs * f, wd = ws * f;
  const long total = static_cast<long>(hd) * wd * C2;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C2) * 2;
    const long pix = i / C2;
    const int x = static_cast<int>(pix % wd), y = static_cast<int>(pix / wd);
    int y0, y1, x0, x1;
    float fy, fx;
    ab_coord(y, f, hs, y0, y1, fy);
    ab_coord(x, f, ws, x0, x1, fx);
    const uint32_t a = *reinterpret_cast<const uint32_t*>(src + (static_cast<long>(y0) * ws + x0) * lds + c);
    const uint32_t b = *reinterpret_cast<const uint32_t*>(src + (static_cast<long>(y0) * ws + x1) * lds + c);
    const uint32_t cc = *reinterpret_cast<const uint32_t*>(src + (static_cast<long>(y1) * ws + x0) * lds + c);
    const uint32_t d = *reinterpret_cast<const uint32_t*>(src + (static_cast<long>(y1) * ws + x1) * lds + c);
    uint32_t* o = reinterpret_cast<uint32_t*>(dst + pix * ldd + c);
    const uint32_t e = *o;
    const float w00 = (1.f - fy) * (1.f - fx), w01 = (1.f - fy) * fx, w10 = fy * (1.f - fx), w11 = fy * fx;
    const float lo = bf16lo(e) + w00 * bf16lo(a) + w01 * bf16lo(b) + w10 * bf16lo(cc) + w11 * bf16lo(d);
    const float hi = bf16hi(e) + w00 * bf16hi(a) + w01 * bf16hi(b) + w10 * bf16hi(cc) + w11 * bf16hi(d);
    *o = pack_bf16(lo, hi);
  }
}

struct MaskLevels {
  const float* dyn[3];  // per level [h*w, ld_dyn] controller outputs of image 0
  long bs[3];           // per level: elements from one image's controller outputs to the next
  int h[3], w[3], stride[3], start[3];
  float soi[3];
};

// Head image b (blockIdx.z) of a batch: its NMS slice is count[b] / anchors + b * bs_anchors, and it reads the mask-branch image
// image_of[b] (image 0 when image_of is null).  Returns -1 when that index is outside [0, S): the image is skipped.
__device__ __forceinline__ int mask_image(const int* __restrict__ image_of, int S) {
  const int img = image_of ? image_of[blockIdx.z] : 0;
  return img >= 0 && img < S ? img : -1;
}

// logits[n, y, x] for instance n (anchor index from the NMS output) — one thread per (instance, pixel)
__global__ void __launch_bounds__(256) mask_logits_kernel(const float* __restrict__ mask_feats, int h, int w, MaskLevels lv, int ld_dyn,
                                                           const int* __restrict__ anchors, long bs_anchors, const int* __restrict__ count,
                                                           const int* __restrict__ image_of, int S, int n_max, float* __restrict__ logits) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  __shared__ float prm[169];
  __shared__ float inst[3];
  const int b = blockIdx.z, img = mask_image(image_of, S);
  if (img < 0) return;
  mask_feats += static_cast<long>(img) * h * w * 8;
  anchors += b * bs_anchors;
  logits += static_cast<long>(b) * n_max * h * w;
  const int n = min(count[b], n_max);
  const int ins = blockIdx.y;
  if (ins >= n) return;
  if (threadIdx.x < 169 || threadIdx.x == 255) {
    const int a = anchors[ins];
    int k = 0;
    if (a >= lv.start[1]) k = 1;
    if (a >= lv.start[2]) k = 2;
    const int ai = a - lv.start[k];
    if (threadIdx.x < 169) prm[threadIdx.x] = lv.dyn[k][b * lv.bs[k] + static_cast<long>(ai) * ld_dyn + threadIdx.x];
    else {
      inst[0] = ((ai % lv.w[k]) + 0.5f) * lv.stride[k];  // locations = (grid + 0.5) * stride (unicorn_head_mask.py:518)
      inst[1] = ((ai / lv.w[k]) + 0.5f) * lv.stride[k];
      inst[2] = lv.soi[k];
    }
  }
  __syncthreads();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= h * w) return;
  float in[10];
  in[0] = (inst[0] - ((pix % w) * 8 + 4)) / inst[2];  // compute_locations: stride 8, + stride // 2 (comm.py:30-45)
  in[1] = (inst[1] - ((pix / w) * 8 + 4)) / inst[2];
  const float4 f0 = *reinterpret_cast<const float4*>(mask_feats + static_cast<long>(pix) * 8);
  const float4 f1 = *reinterpret_cast<const float4*>(mask_feats + static_cast<long>(pix) * 8 + 4);
  in[2] = f0.x; in[3] = f0.y; in[4] = f0.z; in[5] = f0.w; in[6] = f1.x; in[7] = f1.y; in[8] = f1.z; in[9] = f1.w;
  float h1[8], h2[8];
#pragma unroll
  for (int o = 0; o < 8; ++o) {
    float s = prm[152 + o];
#pragma unroll
    for (int i = 0; i < 10; ++i) s += prm[o * 10 + i] * in[i];
    h1[o] = fmaxf(s, 0.f);
  }
#pragma unroll
  for (int o = 0; o < 8; ++o) {
    float s = prm[160 + o];
#pragma unroll
    for (int i = 0; i < 8; ++i) s += prm[80 + o * 8 + i] * h1[i];
    h2[o] = fmaxf(s, 0.f);
  }
  float s = prm[168];
#pragma unroll
  for (int i = 0; i < 8; ++i) s += prm[144 + i] * h2[i];
  logits[static_cast<long>(ins) * h * w + pix] = s;
}

// convex upsampling x up (softmax over the 9 neighbours, weights from up_masks [h,w,9*up*up]) + sigmoid
__global__ void __launch_bounds__(256) mask_convex_up_kernel(const float* __restrict__ logits, const float* __restrict__ up_masks, int h,
                                                              int w, int up, const int* __restrict__ count, const int* __restrict__ image_of,
                                                              int S, int n_max, float* __restrict__ out) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int b = blockIdx.z, img = mask_image(image_of, S);
  if (img < 0) return;
  const int n = min(count[b], n_max);
  const int ins = blockIdx.y;
  if (ins >= n) return;
  const int H = h * up, W = w * up;
  up_masks += static_cast<long>(img) * h * w * (9 * up * up);
  logits += static_cast<long>(b) * n_max * h * w;
  out += static_cast<long>(b) * n_max * H * W;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= H * W) return;
  const int X = t % W, Y = t / W;
  const int x = X / up, y = Y / up, j = X % up, i = Y % up;
  const float* um = up_masks + (static_cast<long>(y) * w + x) * (9 * up * up) + i * up + j;
  float m[9], mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < 9; ++k) { m[k] = um[k * up * up]; mx = fmaxf(mx, m[k]); }
  float den = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) { m[k] = expf(m[k] - mx); den += m[k]; }
  const float* lg = logits + static_cast<long>(ins) * h * w;
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
    const float v = (yy >= 0 && yy < h && xx >= 0 && xx < w) ? lg[yy * w + xx] : 0.f;
    acc += m[k] / den * v;
  }
  out[static_cast<long>(ins) * H * W + t] = 1.f / (1.f + expf(-acc));
}

__global__ void __launch_bounds__(256) mask_final_up_kernel(const float* __restrict__ src, int hs, int ws, int f,
                                                             const int* __restrict__ count, const int* __restrict__ image_of, int S,
                                                             int n_max, float* __restrict__ out) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int b = blockIdx.z;
  if (mask_image(image_of, S) < 0) return;
  const int n = min(count[b], n_max);
  const int ins = blockIdx.y;
  if (ins >= n) return;
  const int hd = hs * f, wd = ws * f;
  src += static_cast<long>(b) * n_max * hs * ws;
  out += static_cast<long>(b) * n_max * hd * wd;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= hd * wd) return;
  int y0, y1, x0, x1;
  float fy, fx;
  ab_coord(t / wd, f, hs, y0, y1, fy);
  ab_coord(t % wd, f, ws, x0, x1, fx);
  const float* s = src + static_cast<long>(ins) * hs * ws;
  out[static_cast<long>(ins) * hd * wd + t] = (1.f - fy) * ((1.f - fx) * s[y0 * ws + x0] + fx * s[y0 * ws + x1]) +
                                             fy * ((1.f - fx) * s[y1 * ws + x0] + fx * s[y1 * ws + x1]);
}


// ------------------------------------------------------------------------------------------------ resize to the original frame
// F.interpolate(m, scale_factor=1/r, mode="bilinear", align_corners=False)[..., :H, :W] of an Hin x Win map, as the VOS and MOTS
// evaluators resize network-resolution masks to the original frame.  PyTorch's output size is floor(in * (1/r)) in double
// precision and its source scale is 1 / (1/r) rounded to float, so the result can be SHORTER than H x W (an 800-row input and a
// 402-row frame give 401 rows): only the hm x wm corner is covered.
struct FrameResize {
  int hm, wm;
  float scale;
};
static FrameResize frame_resize(int Hin, int Win, int H, int W, double r) {
  const double sf = 1.0 / r;
  return FrameResize{std::min(H, static_cast<int>(std::floor(Hin * sf))), std::min(W, static_cast<int>(std::floor(Win * sf))),
                     static_cast<float>(1.0 / sf)};
}
// PyTorch's source index rule (see bilinear_kernel in misc_kernels.cu) for output index i of a source of n samples
__device__ __forceinline__ void resize_src(int i, float scale, int n, int& i0, int& i1, float& l) {
  const float f = fmaxf((i + 0.5f) * scale - 0.5f, 0.f);
  i0 = min(static_cast<int>(f), n - 1);
  i1 = min(i0 + 1, n - 1);
  l = f - i0;
}
__device__ __forceinline__ float resize_sample(const float* s, int ld, int y0, int y1, int x0, int x1, float ly, float lx) {
  return (1.f - ly) * ((1.f - lx) * s[y0 * ld + x0] + lx * s[y0 * ld + x1]) + ly * ((1.f - lx) * s[y1 * ld + x0] + lx * s[y1 * ld + x1]);
}

// ------------------------------------------------------------------------------------------------ VOS soft aggregation
// external/lib/test/tracker/unicorn_vos.py:129-155 (resize of every object's best mask to the original frame:
// F.interpolate(scale_factor=1/r, bilinear, align_corners=False)[:H, :W] into a zero map) and :105-121 (soft aggregation:
// background = prod_i (1 - m_i) in float32 in list order, argmax over [background, m_id...] with the lower channel winning
// ties, label = object id).  One thread per original-frame pixel; the resized soft masks are optional outputs.  blockIdx.y selects
// the video: every video has its own objects, original size, resize and outputs, the network resolution Hin x Win is shared.
constexpr int kVosMaxObj = 16;
constexpr int kVosMaxVideos = UC_VOS_MAX_VIDEOS;
struct VosVideo {
  const float* mask[kVosMaxObj];       // network-resolution soft mask [Hin, Win] or nullptr
  const uint8_t* init_mask[kVosMaxObj];  // original-frame label map [H, W]: object = (label == id), or nullptr
  float* soft;                         // [n, H, W] or nullptr
  uint8_t* seg;                        // [H, W]
  int H, W, hm, wm;                    // original frame, and the corner the resize covers
  float scale;                         // source scale of the resize
  int n;
  uint8_t id[kVosMaxObj];
  uint8_t by_id[kVosMaxObj];  // object indices in ascending id order (argmax tie-breaking)
};
struct VosVideos {
  VosVideo v[kVosMaxVideos];
};
// CUDA 12.1+ guarantees 32764 bytes of kernel parameters on sm_70 and later
static_assert(sizeof(VosVideos) <= 32764, "the VOS descriptors must fit the kernel-parameter block");

__global__ void __launch_bounds__(256) vos_aggregate_kernel(const __grid_constant__ VosVideos vs, int Hin, int Win) {
  pdl_wait();
  pdl_launch_dependents();
  const VosVideo& o = vs.v[blockIdx.y];
  const int H = o.H, W = o.W, hm = o.hm, wm = o.wm;
  const float scale = o.scale;
  float* __restrict__ soft = o.soft;
  uint8_t* __restrict__ seg = o.seg;
  const long total = static_cast<long>(H) * W;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % W), y = static_cast<int>(i / W);
    float m[kVosMaxObj];
    const bool inside = y < hm && x < wm;
    int y0 = 0, y1 = 0, x0 = 0, x1 = 0;
    float ly = 0.f, lx = 0.f;
    if (inside) {
      resize_src(y, scale, Hin, y0, y1, ly);
      resize_src(x, scale, Win, x0, x1, lx);
    }
    float bg = 1.f;
#pragma unroll 1
    for (int k = 0; k < o.n; ++k) {
      float v = 0.f;
      if (o.init_mask[k]) {
        v = o.init_mask[k][i] == static_cast<uint8_t>(o.id[k]) ? 1.f : 0.f;
      } else if (o.mask[k] && inside) {
        v = resize_sample(o.mask[k], Win, y0, y1, x0, x1, ly, lx);
      }
      m[k] = v;
      if (soft) soft[static_cast<long>(k) * total + i] = v;
      bg = bg * (1.f - v);
    }
    float best = bg;
    int label = 0;
#pragma unroll 1
    for (int t = 0; t < o.n; ++t) {
      const int k = o.by_id[t];
      if (m[k] > best) { best = m[k]; label = o.id[k]; }
    }
    seg[i] = static_cast<uint8_t>(label);
  }
}

// ------------------------------------------------------------------------------------------------ MOTS mask encoding
// unicorn/evaluators/mot_evaluator.py:804-805 (resize + threshold), :858-866 (overlap free in ascending track id order against the
// ORIGINAL masks of the earlier instances), :884-888 (COCO compressed RLE of the Fortran-ordered mask, results.rle_encode).
// A mask is a column-major bit sequence of P = hm * wm pixels, stored as 32-bit words that never straddle a column: word
// (x, wy) holds rows 32 wy .. 32 wy + 31 of column x.  The runs start with the zero run, so a run ends at every pixel whose bit
// differs from the previous one (pixel -1 counts as 0) and at P; pass 1 stores exactly those boundary bits.
constexpr int kMotsThreads = 1024;
constexpr int kMotsMaxImages = UC_MOTS_MAX_IMAGES;

struct MotsWs {
  uint32_t* diff;      // run boundaries of the emitted instances, [k_b][words_b] per image, the images one after another
  int4* state;         // [k][kMotsThreads] run state before each thread's chunk of words
  int* char_off;       // [k][kMotsThreads] chars before each thread's chunk, within the instance
  long long* nchars;   // [k] chars of each instance (0 when not emitted)
};
static inline long align16(long b) { return (b + 15) & ~15L; }
// k instances in all, diff_words boundary words in all
static long mots_workspace_bytes(int k, long diff_words) {
  return align16(4L * diff_words) + align16(16L * k * kMotsThreads) + align16(4L * k * kMotsThreads) + align16(8L * k);
}
static MotsWs mots_ws(void* base, int k, long diff_words) {
  char* p = static_cast<char*>(base);
  MotsWs w;
  w.diff = reinterpret_cast<uint32_t*>(p);
  p += align16(4L * diff_words);
  w.state = reinterpret_cast<int4*>(p);
  p += align16(16L * k * kMotsThreads);
  w.char_off = reinterpret_cast<int*>(p);
  p += align16(4L * k * kMotsThreads);
  w.nchars = reinterpret_cast<long long*>(p);
  return w;
}

// The images of one encode, passed by value: image b owns instances [k0[b], k0[b + 1]) of the flat order / emit lists, its masks
// are resized to hm[b] x wm[b] with source scale[b], and instance j of it keeps its boundary words at
// diff0[b] + (j - k0[b]) * wm[b] * ceil(hm[b] / 32) in MotsWs::diff.
struct MotsImages {
  int n;
  int k0[kMotsMaxImages + 1];
  int hm[kMotsMaxImages], wm[kMotsMaxImages];
  float scale[kMotsMaxImages];
  long diff0[kMotsMaxImages];
};
// The resized size and boundary words of instance j's image; returns the instance's boundary words.
__device__ __forceinline__ const uint32_t* mots_instance(const MotsImages& im, const MotsWs& ws, int j, int& hm, int& wm, int& hw32,
                                                         long& words) {
  int b = 0;
  while (j >= im.k0[b + 1]) ++b;
  hm = im.hm[b];
  wm = im.wm[b];
  hw32 = (hm + 31) / 32;
  words = static_cast<long>(wm) * hw32;
  return ws.diff + im.diff0[b] + (j - im.k0[b]) * words;
}

// Pass 1: one thread per word of image blockIdx.z, looping over the image's instances in `order`; the 32 lanes of a warp take 32
// neighbouring columns of the same rows, so their bilinear taps share source rows.  The pixel before the word is resampled too, so
// the boundary bits of the word need no neighbour.
__global__ void __launch_bounds__(256) mots_planes_kernel(const float* __restrict__ masks, long bs_masks, int n_max, int Hin, int Win,
                                                          const int* __restrict__ order, const uint8_t* __restrict__ emit, float thr,
                                                          const __grid_constant__ MotsImages im, MotsWs ws) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.z, hm = im.hm[b], wm = im.wm[b];
  const float scale = im.scale[b];
  const int x = blockIdx.x * 32 + threadIdx.x, wy = blockIdx.y * 8 + threadIdx.y, hw32 = (hm + 31) / 32;
  if (x >= wm || wy >= hw32) return;
  const long words = static_cast<long>(wm) * hw32;
  masks += b * bs_masks;
  const int j0 = im.k0[b], j1 = im.k0[b + 1];
  uint32_t* diff = ws.diff + im.diff0[b];
  int x0, x1;
  float lx;
  resize_src(x, scale, Win, x0, x1, lx);
  const bool has_prev = wy > 0 || x > 0;  // the pixel before this word in column-major order
  int py0 = 0, py1 = 0, px0 = 0, px1 = 0;
  float ply = 0.f, plx = 0.f;
  if (has_prev) {
    resize_src(wy > 0 ? 32 * wy - 1 : hm - 1, scale, Hin, py0, py1, ply);
    resize_src(wy > 0 ? x : x - 1, scale, Win, px0, px1, plx);
  }
  const int ybase = 32 * wy, nrows = min(32, hm - ybase);
  const uint32_t valid = nrows == 32 ? ~0u : (1u << nrows) - 1u;
  uint32_t acc = 0, accp = 0;  // pixels claimed by the original masks of the earlier instances
#pragma unroll 1
  for (int j = j0; j < j1; ++j) {
    const int row = order[j];
    uint32_t raw = 0, rawp = 0;
    if (row >= 0 && row < n_max) {  // a row outside the mask buffer reads as an empty mask
      const float* s = masks + static_cast<long>(row) * Hin * Win;
#pragma unroll 4
      for (int r = 0; r < nrows; ++r) {
        int y0, y1;
        float ly;
        resize_src(ybase + r, scale, Hin, y0, y1, ly);
        raw |= static_cast<uint32_t>(resize_sample(s, Win, y0, y1, x0, x1, ly, lx) > thr) << r;
      }
      if (has_prev) rawp = resize_sample(s, Win, py0, py1, px0, px1, ply, plx) > thr;
    }
    const uint32_t fr = raw & ~acc, frp = rawp & ~accp;
    acc |= raw;
    accp |= rawp;
    if (emit[j]) diff[(j - j0) * words + static_cast<long>(x) * hw32 + wy] = (fr ^ ((fr << 1) | frp)) & valid;
  }
}

// ------------------------------------------------------------------------------------------------ COCO instance encoding
// COCOInstEvaluator.convert_to_coco_format (unicorn/evaluators/coco_inst_evaluator.py): every NMS row's mask
// aligned_bilinear(x f)-upsampled to the network input (utils/boxes.py:138-145), resized by 1/r to the original frame
// (F.interpolate(scale_factor=1/r, bilinear)[:, 0, :H, :W]) and thresholded, without writing the full-resolution mask.  The encoded
// mask is the whole H x W frame: pixels outside the hm x wm corner the resize produces are background.
//
// The sample of mask_final_up_kernel at full-resolution pixel (Y, X), with the operation order nvcc gives that kernel (its SASS:
// one product per source row, fused with the other column's term, then the rows the same way): bit-identical to what it stores.
// fy == 0 (every other row at f = 2, the same for the whole warp) skips the second source row: the maps are sigmoid outputs in
// [0, 1], so fma(1, top, 0 * bot) == top exactly.
__device__ __forceinline__ float final_up_at(const float* __restrict__ s, int ws, int y0, int y1, float fy, int x0, int x1, float fx) {
  const float gx = 1.f - fx;
  const float top = __fmaf_rn(fx, s[y0 * ws + x1], __fmul_rn(gx, s[y0 * ws + x0]));
  if (fy == 0.f) return top;
  const float bot = __fmaf_rn(fx, s[y1 * ws + x1], __fmul_rn(gx, s[y1 * ws + x0]));
  return __fmaf_rn(1.f - fy, top, __fmul_rn(fy, bot));
}
// resize_sample's order of operations in mots_planes_kernel (its SASS), on the four taps of the resize
__device__ __forceinline__ float resize_mix(float a, float b, float c, float d, float ly, float lx) {
  const float gx = 1.f - lx;
  const float top = __fmaf_rn(gx, a, __fmul_rn(lx, b));
  const float bot = __fmaf_rn(gx, c, __fmul_rn(lx, d));
  return __fmaf_rn(1.f - ly, top, __fmul_rn(ly, bot));
}
// The aligned_bilinear taps of the two full-resolution indices i0, i1 the resize reads.
struct AbTaps {
  int a0, a1, b0, b1;
  float fa, fb;
};
// ab_coord's taps; for a power-of-two f the fraction k / f is exact, so k * (1 / f) is the same float without the division.
__device__ __forceinline__ void ab_coord_fast(int i, int f, float inv_f, int n, int& i0, int& i1, float& frac) {
  if (inv_f == 0.f) {
    ab_coord(i, f, n, i0, i1, frac);
    return;
  }
  const int ii = max(i - f / 2, 0);
  i0 = ii / f;
  frac = static_cast<float>(ii - i0 * f) * inv_f;
  i1 = min(i0 + 1, n - 1);
  i0 = min(i0, n - 1);
}
__device__ __forceinline__ AbTaps ab_taps(int i0, int i1, int f, float inv_f, int n) {
  AbTaps t;
  ab_coord_fast(i0, f, inv_f, n, t.a0, t.a1, t.fa);
  ab_coord_fast(i1, f, inv_f, n, t.b0, t.b1, t.fb);
  return t;
}
// The resized, upsampled mask at original-frame pixel (y, x) of the column taps tx (x resized to lx).
__device__ __forceinline__ float inst_sample(const float* __restrict__ s, int hs, int ws, int f, float inv_f, int Hin, float scale, int y,
                                            const AbTaps& tx, float lx) {
  int Y0, Y1;
  float ly;
  resize_src(y, scale, Hin, Y0, Y1, ly);
  const AbTaps ty = ab_taps(Y0, Y1, f, inv_f, hs);
  return resize_mix(final_up_at(s, ws, ty.a0, ty.a1, ty.fa, tx.a0, tx.a1, tx.fa), final_up_at(s, ws, ty.a0, ty.a1, ty.fa, tx.b0, tx.b1, tx.fb),
                    final_up_at(s, ws, ty.b0, ty.b1, ty.fb, tx.a0, tx.a1, tx.fa), final_up_at(s, ws, ty.b0, ty.b1, ty.fb, tx.b0, tx.b1, tx.fb),
                    ly, lx);
}

// The part of each image's H x W frame the resize covers (rows < hv, columns < wv).
struct InstCover {
  int hv[kMotsMaxImages], wv[kMotsMaxImages];
};

// Pass 1 of the instance encode: slot j = blockIdx.z (image b = j / n_max, row row0 + j % n_max of its NMS output) is emitted when
// that row exists (count[b] on the device); one thread per word of the slot's H x W frame, as in mots_planes_kernel, with no state
// between instances.  maps: the d_rate = 1 output of uc_dynamic_masks_batched, [B, n_max, hs, ws] (image b at b * bs_maps).
__global__ void __launch_bounds__(256) inst_planes_kernel(const float* __restrict__ maps, long bs_maps, int n_max, int hs, int ws, int f,
                                                          const int* __restrict__ count, int row0, float thr,
                                                          const __grid_constant__ MotsImages im, const __grid_constant__ InstCover cv,
                                                          MotsWs wsp, uint8_t* __restrict__ emit) {
  pdl_wait();
  pdl_launch_dependents();
  const int j = blockIdx.z, b = j / n_max, i = j - b * n_max;
  const bool on = i < count[b] - row0;
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && threadIdx.y == 0) emit[j] = on;
  if (!on) return;
  const int H = im.hm[b], W = im.wm[b], hv = cv.hv[b], wv = cv.wv[b];
  const float scale = im.scale[b];
  const int x = blockIdx.x * 32 + threadIdx.x, wy = blockIdx.y * 8 + threadIdx.y, hw32 = (H + 31) / 32;
  if (x >= W || wy >= hw32) return;
  const int Hin = hs * f, Win = ws * f;
  const float inv_f = (f & (f - 1)) == 0 ? 1.f / f : 0.f;  // 0: divide
  const float* s = maps + b * bs_maps + static_cast<long>(i) * hs * ws;
  AbTaps tx{}, tp{};
  float lx = 0.f, lp = 0.f;
  if (x < wv) {
    int X0, X1;
    resize_src(x, scale, Win, X0, X1, lx);
    tx = ab_taps(X0, X1, f, inv_f, ws);
  }
  // the pixel before this word in column-major order: row 32 wy - 1 of column x, or the last row of column x - 1
  const int py = wy > 0 ? 32 * wy - 1 : H - 1, px = wy > 0 ? x : x - 1;
  const bool prev_in = px >= 0 && px < wv && py < hv;
  if (prev_in && px != x) {
    int X0, X1;
    resize_src(px, scale, Win, X0, X1, lp);
    tp = ab_taps(X0, X1, f, inv_f, ws);
  } else if (prev_in) {
    tp = tx;
    lp = lx;
  }
  const int ybase = 32 * wy, nrows = min(32, H - ybase);
  const uint32_t valid = nrows == 32 ? ~0u : (1u << nrows) - 1u;
  uint32_t raw = 0;
  if (x < wv) {
    const int rows = min(nrows, hv - ybase);
#pragma unroll 4
    for (int r = 0; r < rows; ++r) raw |= static_cast<uint32_t>(inst_sample(s, hs, ws, f, inv_f, Hin, scale, ybase + r, tx, lx) > thr) << r;
  }
  const uint32_t rawp = prev_in ? inst_sample(s, hs, ws, f, inv_f, Hin, scale, py, tp, lp) > thr : 0u;
  wsp.diff[im.diff0[b] + static_cast<long>(i) * W * hw32 + static_cast<long>(x) * hw32 + wy] = (raw ^ ((raw << 1) | rawp)) & valid;
}

// Run state after a prefix of the boundaries: their number and the last three boundary positions (-1: none).
__device__ __forceinline__ int4 run_push(int4 s, int pos) { return make_int4(s.x + 1, pos, s.y, s.z); }
__device__ __forceinline__ int4 run_cat(int4 a, int4 b) {
  if (b.x >= 3) return make_int4(a.x + b.x, b.y, b.z, b.w);
  if (b.x == 2) return make_int4(a.x + 2, b.y, b.z, a.y);
  if (b.x == 1) return make_int4(a.x + 1, b.y, a.y, a.z);
  return a;
}
// The COCO count that ends at `pos`, minus the count two before it (rleToString: "if (i > 2) x -= cnts[i - 2]").
__device__ __forceinline__ int run_delta(int4 s, int pos) {
  const int c = pos - (s.x >= 1 ? s.y : 0);
  return s.x > 2 ? c - (s.z - s.w) : c;  // count i - 2 spans boundaries i - 3 .. i - 2
}
// 5 data bits per char with a continuation bit, +48; writes the chars below `cap` when out != nullptr, returns their number.
__device__ __forceinline__ int rle_chars(int x, char* out, long long off, long cap) {
  int n = 0;
  bool more = true;
  while (more) {
    int c = x & 0x1f;
    x >>= 5;
    more = (c & 0x10) ? x != -1 : x != 0;
    if (more) c |= 0x20;
    if (out && off + n < cap) out[off + n] = static_cast<char>(c + 48);
    ++n;
  }
  return n;
}

template <typename T, typename Op>
__device__ T block_exclusive_scan(T v, T identity, Op op, T* sh, T& total) {
  const int t = threadIdx.x, n = blockDim.x;
  sh[t] = v;
  __syncthreads();
  for (int o = 1; o < n; o <<= 1) {
    const T a = t >= o ? sh[t - o] : identity;
    __syncthreads();
    if (t >= o) sh[t] = op(a, sh[t]);
    __syncthreads();
  }
  const T excl = t > 0 ? sh[t - 1] : identity;
  total = sh[n - 1];
  __syncthreads();
  return excl;
}

// Walks the boundaries of words [w0, w1) of one instance from run state s; f(pos, s) sees the state before each boundary.
template <typename F>
__device__ __forceinline__ int4 mots_walk(const uint32_t* __restrict__ d, long w0, long w1, int hm, int hw32, int4 s, F f) {
  for (long w = w0; w < w1; ++w) {
    uint32_t bits = d[w];
    if (!bits) continue;
    const int x = static_cast<int>(w / hw32), wy = static_cast<int>(w - static_cast<long>(x) * hw32);
    const int base = x * hm + 32 * wy;
    while (bits) {
      const int pos = base + __ffs(bits) - 1;
      bits &= bits - 1;
      f(pos, s);
      s = run_push(s, pos);
    }
  }
  return s;
}

// Pass 2: one block per instance of any image; each thread owns a contiguous chunk of words.  Scan of the run states over the
// chunks, then the number of chars of every count, scanned into each chunk's char offset.
__global__ void __launch_bounds__(kMotsThreads) mots_runs_kernel(const uint8_t* __restrict__ emit, const __grid_constant__ MotsImages im,
                                                                 MotsWs ws) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ int4 sh_state[kMotsThreads];
  __shared__ long long sh_chars[kMotsThreads];
  const int j = blockIdx.x, t = threadIdx.x;
  if (!emit[j]) {
    if (t == 0) ws.nchars[j] = 0;
    return;
  }
  int hm, wm, hw32;
  long words;
  const uint32_t* d = mots_instance(im, ws, j, hm, wm, hw32, words);
  const long chunk = (words + kMotsThreads - 1) / kMotsThreads;
  const long w0 = std::min(words, t * chunk), w1 = std::min(words, w0 + chunk);
  const int4 none = make_int4(0, -1, -1, -1);
  const int4 mine = mots_walk(d, w0, w1, hm, hw32, none, [](int, int4) {});
  int4 all;
  const int4 pre = block_exclusive_scan(mine, none, [](int4 a, int4 b) { return run_cat(a, b); }, sh_state, all);
  ws.state[static_cast<long>(j) * kMotsThreads + t] = pre;
  long long n = 0;
  mots_walk(d, w0, w1, hm, hw32, pre, [&](int pos, int4 s) { n += rle_chars(run_delta(s, pos), nullptr, 0, 0); });
  if (t == kMotsThreads - 1) n += rle_chars(run_delta(all, hm * wm), nullptr, 0, 0);  // the last run ends at P
  long long total;
  const long long off = block_exclusive_scan(n, 0LL, [](long long a, long long b) { return a + b; }, sh_chars, total);
  ws.char_off[static_cast<long>(j) * kMotsThreads + t] = static_cast<int>(off);
  if (t == 0) ws.nchars[j] = total;
}

// Pass 3: the offsets of the k strings of all images (block 0) and the chars of every emitted instance (block j), clipped at the
// capacity.
__global__ void __launch_bounds__(kMotsThreads) mots_chars_kernel(const uint8_t* __restrict__ emit, const __grid_constant__ MotsImages im,
                                                                  MotsWs ws, char* __restrict__ chars, long capacity,
                                                                  long long* __restrict__ offsets) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ long long base;
  const int j = blockIdx.x, t = threadIdx.x, k = im.k0[im.n];
  if (t == 0) {
    long long b = 0;
    for (int i = 0; i < k; ++i) {
      if (j == 0) offsets[i] = b;
      if (i == j) base = b;
      b += ws.nchars[i];
    }
    if (j == 0) offsets[k] = b;
  }
  __syncthreads();
  if (j >= k || !emit[j]) return;
  int hm, wm, hw32;
  long words;
  const uint32_t* d = mots_instance(im, ws, j, hm, wm, hw32, words);
  const long chunk = (words + kMotsThreads - 1) / kMotsThreads;
  const long w0 = std::min(words, t * chunk), w1 = std::min(words, w0 + chunk);
  long long off = base + ws.char_off[static_cast<long>(j) * kMotsThreads + t];
  const int4 end = mots_walk(d, w0, w1, hm, hw32, ws.state[static_cast<long>(j) * kMotsThreads + t],
                             [&](int pos, int4 s) { off += rle_chars(run_delta(s, pos), chars, off, capacity); });
  if (t == kMotsThreads - 1) rle_chars(run_delta(end, hm * wm), chars, off, capacity);
}

// B images; the batched entry points validate every argument before any CUDA call, with errors prefixed by `what`.
static int aligned_bilinear_add(const char* what, const void* src, int lds, long bs_src, int hs, int ws, void* dst, int ldd, long bs_dst, int C,
                                int factor, int B, cudaStream_t stream) {
  if (!src || !dst) return set_error(UC_EINVAL, "%s: null pointer", what);
  if (B < 1) return set_error(UC_EINVAL, "%s: B must be >= 1 (got %d)", what, B);
  if (C % 2 || lds % 2 || ldd % 2 || factor < 1 || hs < 1 || ws < 1 || lds < C || ldd < C) return set_error(UC_EINVAL, "%s: bad arguments", what);
  const long src_img = static_cast<long>(hs) * ws * lds, dst_img = static_cast<long>(hs) * factor * ws * factor * ldd;
  if (bs_src % 2 || bs_dst % 2 || bs_src < src_img || bs_dst < dst_img)
    return set_error(UC_EINVAL, "%s: bad per-image strides (even, src >= hs*ws*lds = %ld, dst >= (hs*f)*(ws*f)*ldd = %ld)", what, src_img, dst_img);
  const long total = static_cast<long>(hs) * factor * ws * factor * (C / 2);
  const long cap = std::max<long>(1, static_cast<long>(num_sms()) * 16 / B);  // the whole batch keeps the B = 1 launch's CTA budget
  const int grid = static_cast<int>(std::max<long>(1, std::min<long>((total + 255) / 256, cap)));
  launch_pdl(aligned_bilinear_add_kernel, dim3(grid, B), 256, 0, stream, static_cast<const uint16_t*>(src), lds, bs_src, hs, ws,
             static_cast<uint16_t*>(dst), ldd, bs_dst, C, factor);
  return check_launch(what);
}

static int dynamic_masks(const char* what, const float* mask_feats, const float* up_masks, int S, int h, int w, int up_rate, int d_rate,
                         const float* const* dyn_levels, int ld_dyn, const long* bs_dyn, const int* level_hw, const int* level_strides,
                         const float* level_soi, const int* anchors_dev, long bs_anchors, const int* count_dev, const int* image_of, int B,
                         int n_max, float* scratch, float* out_masks, cudaStream_t stream) {
  if (!mask_feats || !up_masks || !dyn_levels || !level_hw || !level_strides || !level_soi || !anchors_dev || !count_dev || !scratch || !out_masks)
    return set_error(UC_EINVAL, "%s: null pointer", what);
  if (B < 1) return set_error(UC_EINVAL, "%s: B must be >= 1 (got %d)", what, B);
  if (S < 1) return set_error(UC_EINVAL, "%s: S (mask-branch images) must be >= 1 (got %d)", what, S);
  if (n_max < 1 || ld_dyn < 169 || up_rate < 1 || d_rate < 1 || h < 1 || w < 1) return set_error(UC_EINVAL, "%s: bad sizes", what);
  if (B > 65535 || n_max > 65535) return set_error(UC_EINVAL, "%s: B and n_max must be <= 65535", what);
  MaskLevels lv;
  int start = 0;
  for (int k = 0; k < 3; ++k) {
    if (!dyn_levels[k]) return set_error(UC_EINVAL, "%s: null pointer", what);
    lv.dyn[k] = dyn_levels[k];
    lv.h[k] = level_hw[2 * k]; lv.w[k] = level_hw[2 * k + 1]; lv.stride[k] = level_strides[k]; lv.soi[k] = level_soi[k];
    lv.bs[k] = bs_dyn ? bs_dyn[k] : 0;
    lv.start[k] = start;
    start += lv.h[k] * lv.w[k];
    if (bs_dyn && lv.bs[k] < static_cast<long>(lv.h[k]) * lv.w[k] * ld_dyn)
      return set_error(UC_EINVAL, "%s: bad per-image strides of level %d (controller outputs: >= h*w*ld_dyn = %ld)", what, k,
                       static_cast<long>(lv.h[k]) * lv.w[k] * ld_dyn);
  }
  if (bs_dyn && bs_anchors < start) return set_error(UC_EINVAL, "%s: bad per-image anchor stride %ld (>= %d anchors)", what, bs_anchors, start);
  float* logits = scratch;                                       // [B, n_max, h, w]
  float* mid = scratch + static_cast<long>(B) * n_max * h * w;    // [B, n_max, h*up, w*up]
  launch_pdl(mask_logits_kernel, dim3((h * w + 255) / 256, n_max, B), 256, 0, stream, mask_feats, h, w, lv, ld_dyn, anchors_dev, bs_anchors,
             count_dev, image_of, S, n_max, logits);
  const int H1 = h * up_rate, W1 = w * up_rate;
  launch_pdl(mask_convex_up_kernel, dim3((H1 * W1 + 255) / 256, n_max, B), 256, 0, stream, logits, up_masks, h, w, up_rate, count_dev, image_of,
             S, n_max, d_rate == 1 ? out_masks : mid);
  if (d_rate != 1) {
    const int H2 = H1 * d_rate, W2 = W1 * d_rate;
    launch_pdl(mask_final_up_kernel, dim3((H2 * W2 + 255) / 256, n_max, B), 256, 0, stream, mid, H1, W1, d_rate, count_dev, image_of, S, n_max,
               out_masks);
  }
  return check_launch(what);
}

}  // namespace uc

using namespace uc;

extern "C" int uc_aligned_bilinear_add(const void* src, int lds, int hs, int ws, void* dst, int ldd, int C, int factor, void* stream_v) {
  if (!src || !dst || C % 2 || lds % 2 || ldd % 2 || factor < 1) return set_error(UC_EINVAL, "uc_aligned_bilinear_add: bad arguments");
  return aligned_bilinear_add("uc_aligned_bilinear_add", src, lds, static_cast<long>(hs) * ws * lds, hs, ws, dst, ldd,
                              static_cast<long>(hs) * factor * ws * factor * ldd, C, factor, 1, static_cast<cudaStream_t>(stream_v));
}

extern "C" int uc_aligned_bilinear_add_batched(const void* src, int lds, long bs_src, int hs, int ws, void* dst, int ldd, long bs_dst, int C,
                                               int factor, int B, void* stream_v) {
  return aligned_bilinear_add("uc_aligned_bilinear_add_batched", src, lds, bs_src, hs, ws, dst, ldd, bs_dst, C, factor, B,
                              static_cast<cudaStream_t>(stream_v));
}

extern "C" int uc_dynamic_masks(const float* mask_feats, const float* up_masks, int h, int w, int up_rate, int d_rate,
                                const float* const* dyn_levels, int ld_dyn, const int* level_hw, const int* level_strides,
                                const float* level_soi, const int* anchors_dev, const int* count_dev, int n_max, float* scratch,
                                float* out_masks, void* stream_v) {
  return dynamic_masks("uc_dynamic_masks", mask_feats, up_masks, 1, h, w, up_rate, d_rate, dyn_levels, ld_dyn, nullptr, level_hw, level_strides,
                       level_soi, anchors_dev, 0, count_dev, nullptr, 1, n_max, scratch, out_masks, static_cast<cudaStream_t>(stream_v));
}

extern "C" int uc_dynamic_masks_batched(const float* mask_feats, const float* up_masks, int S, int h, int w, int up_rate, int d_rate,
                                        const float* const* dyn_levels, int ld_dyn, const long* bs_dyn, const int* level_hw,
                                        const int* level_strides, const float* level_soi, const int* anchors_dev, long bs_anchors,
                                        const int* count_dev, const int* image_of, int B, int n_max, float* scratch, float* out_masks,
                                        void* stream_v) {
  if (!bs_dyn || !image_of) return set_error(UC_EINVAL, "uc_dynamic_masks_batched: null pointer (bs_dyn and image_of are required)");
  return dynamic_masks("uc_dynamic_masks_batched", mask_feats, up_masks, S, h, w, up_rate, d_rate, dyn_levels, ld_dyn, bs_dyn, level_hw,
                       level_strides, level_soi, anchors_dev, bs_anchors, count_dev, image_of, B, n_max, scratch, out_masks,
                       static_cast<cudaStream_t>(stream_v));
}

// The assembly of B videos in one launch (B = 1: uc_vos_aggregate).  Every argument is validated before any CUDA call, with errors
// prefixed by `what`, and by the video when the call is batched.
static int vos_aggregate(const char* what, bool batched, const UcVosVideo* videos, int B, int Hin, int Win, cudaStream_t stream) {
  if (!videos) return set_error(UC_EINVAL, "%s: null pointer", what);
  if (B < 1 || B > kVosMaxVideos) return set_error(UC_EINVAL, "%s: B = %d must be in 1..%d", what, B, kVosMaxVideos);
  char at[96];
  VosVideos vs;
  memset(&vs, 0, sizeof(vs));
  long total_max = 0;
  for (int b = 0; b < B; ++b) {
    if (batched) snprintf(at, sizeof(at), "%s: video %d", what, b);
    else snprintf(at, sizeof(at), "%s", what);
    const UcVosVideo& in = videos[b];
    if (!in.objs || !in.seg_out || in.n < 1 || in.n > kVosMaxObj) return set_error(UC_EINVAL, "%s: 1..%d objects", at, kVosMaxObj);
    if (Hin < 1 || Win < 1 || in.H < 1 || in.W < 1 || !(in.r > 0.f)) return set_error(UC_EINVAL, "%s: bad sizes", at);
    VosVideo& o = vs.v[b];
    o.n = in.n;
    for (int k = 0; k < in.n; ++k) {
      if (in.objs[k].id < 1 || in.objs[k].id > 255) return set_error(UC_EINVAL, "%s: object ids must be 1..255", at);
      o.mask[k] = in.objs[k].mask; o.init_mask[k] = in.objs[k].init_mask; o.id[k] = static_cast<uint8_t>(in.objs[k].id);
      o.by_id[k] = static_cast<uint8_t>(k);
    }
    std::stable_sort(o.by_id, o.by_id + in.n, [&](int a, int c) { return o.id[a] < o.id[c]; });
    const FrameResize rs = frame_resize(Hin, Win, in.H, in.W, in.r);
    o.H = in.H; o.W = in.W; o.hm = rs.hm; o.wm = rs.wm; o.scale = rs.scale;
    o.soft = in.soft_out;
    o.seg = in.seg_out;
    total_max = std::max(total_max, static_cast<long>(in.H) * in.W);
  }
  // the x dimension stride-loops over the largest frame; a CTA past its own video's pixels does nothing
  const int grid = static_cast<int>(std::max<long>(1, std::min<long>((total_max + 255) / 256, static_cast<long>(num_sms()) * 16)));
  launch_pdl(vos_aggregate_kernel, dim3(grid, B), 256, 0, stream, vs, Hin, Win);
  return check_launch(what);
}

extern "C" int uc_vos_aggregate(const UcVosObject* objs, int n, int Hin, int Win, int H, int W, float r, float* soft_out, uint8_t* seg_out,
                                void* stream_v) {
  const UcVosVideo v{objs, n, H, W, r, soft_out, seg_out};
  return vos_aggregate("uc_vos_aggregate", false, &v, 1, Hin, Win, static_cast<cudaStream_t>(stream_v));
}

extern "C" int uc_vos_aggregate_batched(const UcVosVideo* videos, int B, int Hin, int Win, void* stream_v) {
  return vos_aggregate("uc_vos_aggregate_batched", true, videos, B, Hin, Win, static_cast<cudaStream_t>(stream_v));
}

// One encode over the instances of B images (B = 1: uc_mots_encode).  Every argument is validated before any CUDA call, with errors
// prefixed by `what`, and by the image when the call is batched.
static int mots_encode(const char* what, bool batched, const float* masks, long bs_masks, int n_max, int Hin, int Win, int B, const int* k,
                       const int* H, const int* W, const double* r, const int* order, const uint8_t* emit, float thr, void* workspace,
                       long workspace_bytes, char* chars, long capacity, long long* offsets, cudaStream_t stream) {
  if (!k || !H || !W || !r) return set_error(UC_EINVAL, "%s: null pointer", what);
  if (B < 1 || B > kMotsMaxImages) return set_error(UC_EINVAL, "%s: B = %d must be in 1..%d", what, B, kMotsMaxImages);
  long K = 0;
  for (int b = 0; b < B; ++b) K += std::max(k[b], 0);
  if (K > INT_MAX) return set_error(UC_EINVAL, "%s: more than %d instances", what, INT_MAX);
  if (!masks || !order || !emit || !offsets || (K > 0 && !workspace) || (capacity > 0 && !chars))
    return set_error(UC_EINVAL, "%s: null pointer", what);
  char at[96];
  auto image = [&](int b) {
    if (batched) snprintf(at, sizeof(at), "%s: image %d", what, b);
    else snprintf(at, sizeof(at), "%s", what);
    return at;
  };
  if (n_max < 1 || Hin < 1 || Win < 1) return set_error(UC_EINVAL, "%s: bad sizes", what);
  if (bs_masks < static_cast<long>(n_max) * Hin * Win)
    return set_error(UC_EINVAL, "%s: bad per-image stride %ld (>= n_max*Hin*Win = %ld)", what, bs_masks, static_cast<long>(n_max) * Hin * Win);
  for (int b = 0; b < B; ++b)
    if (H[b] < 1 || W[b] < 1 || !(r[b] > 0.0)) return set_error(UC_EINVAL, "%s: bad sizes", image(b));
  for (int b = 0; b < B; ++b)
    if (k[b] < 0 || k[b] > n_max) return set_error(UC_EINVAL, "%s: k = %d must be in 0..n_max (%d)", image(b), k[b], n_max);
  if (capacity < 0) return set_error(UC_EINVAL, "%s: negative capacity", what);
  if ((reinterpret_cast<uintptr_t>(masks) | reinterpret_cast<uintptr_t>(order)) % 4 || reinterpret_cast<uintptr_t>(offsets) % 8 ||
      reinterpret_cast<uintptr_t>(workspace) % 16)
    return set_error(UC_EINVAL, "%s: masks / order must be 4-byte, offsets 8-byte, workspace 16-byte aligned", what);
  MotsImages im;
  im.n = B;
  im.k0[0] = 0;
  long diff_words = 0;
  int wm_max = 0, hw32_max = 0;
  for (int b = 0; b < B; ++b) {
    const FrameResize rs = frame_resize(Hin, Win, H[b], W[b], r[b]);
    if (rs.hm < 1 || rs.wm < 1) return set_error(UC_EINVAL, "%s: the resized mask is empty (r too large)", image(b));
    const int hw32 = (rs.hm + 31) / 32;
    const long words = static_cast<long>(rs.wm) * hw32;
    if (words > (1L << 31) / 32) return set_error(UC_EINVAL, "%s: frame too large", image(b));
    im.k0[b + 1] = im.k0[b] + k[b];
    im.hm[b] = rs.hm;
    im.wm[b] = rs.wm;
    im.scale[b] = rs.scale;
    im.diff0[b] = diff_words;
    diff_words += k[b] * words;
    wm_max = std::max(wm_max, rs.wm);
    hw32_max = std::max(hw32_max, hw32);
  }
  if (workspace_bytes < mots_workspace_bytes(static_cast<int>(K), diff_words)) return set_error(UC_EINVAL, "%s: workspace too small", what);
  MotsWs ws = mots_ws(workspace, static_cast<int>(K), diff_words);
  if (K > 0) {
    launch_pdl(mots_planes_kernel, dim3((wm_max + 31) / 32, (hw32_max + 7) / 8, B), dim3(32, 8), 0, stream, masks, bs_masks, n_max, Hin, Win,
               order, emit, thr, im, ws);
    launch_pdl(mots_runs_kernel, static_cast<int>(K), kMotsThreads, 0, stream, emit, im, ws);
  }
  launch_pdl(mots_chars_kernel, std::max(static_cast<int>(K), 1), kMotsThreads, 0, stream, emit, im, ws, chars, capacity, offsets);
  return check_launch(what);
}

extern "C" long uc_mots_encode_workspace_bytes(int k_max, int H, int W) {
  if (k_max < 0 || H < 1 || W < 1) return -1;
  return mots_workspace_bytes(k_max, static_cast<long>(k_max) * W * ((H + 31) / 32));
}

extern "C" int uc_mots_encode(const float* masks, int n_max, int Hin, int Win, const int* order, const uint8_t* emit, int k, float thr,
                              double r, int H, int W, void* workspace, long workspace_bytes, char* chars, long capacity,
                              long long* offsets, void* stream_v) {
  return mots_encode("uc_mots_encode", false, masks, static_cast<long>(std::max(n_max, 0)) * std::max(Hin, 0) * std::max(Win, 0), n_max, Hin,
                     Win, 1, &k, &H, &W, &r, order, emit, thr, workspace, workspace_bytes, chars, capacity, offsets,
                     static_cast<cudaStream_t>(stream_v));
}

extern "C" int uc_mots_encode_batched(const float* masks, long bs_masks, int n_max, int Hin, int Win, int B, const int* k, const int* H,
                                      const int* W, const double* r, const int* order, const uint8_t* emit, float thr, void* workspace,
                                      long workspace_bytes, char* chars, long capacity, long long* offsets, void* stream_v) {
  return mots_encode("uc_mots_encode_batched", true, masks, bs_masks, n_max, Hin, Win, B, k, H, W, r, order, emit, thr, workspace,
                     workspace_bytes, chars, capacity, offsets, static_cast<cudaStream_t>(stream_v));
}

extern "C" int uc_inst_encode_batched(const float* maps, long bs_maps, int n_max, int hs, int ws, int d_rate, int B, const int* count_dev,
                                      int row0, const int* H, const int* W, const double* r, float thr, void* workspace,
                                      long workspace_bytes, uint8_t* emit, char* chars, long capacity, long long* offsets, void* stream_v) {
  const char* what = "uc_inst_encode_batched";
  if (!H || !W || !r) return set_error(UC_EINVAL, "%s: null pointer", what);
  if (B < 1 || B > kMotsMaxImages) return set_error(UC_EINVAL, "%s: B = %d must be in 1..%d", what, B, kMotsMaxImages);
  if (!maps || !count_dev || !workspace || !emit || !offsets || (capacity > 0 && !chars)) return set_error(UC_EINVAL, "%s: null pointer", what);
  if (n_max < 1 || hs < 1 || ws < 1 || d_rate < 1) return set_error(UC_EINVAL, "%s: bad sizes", what);
  if (static_cast<long>(B) * n_max > 65535) return set_error(UC_EINVAL, "%s: B * n_max = %ld slots must be <= 65535", what, static_cast<long>(B) * n_max);
  if (row0 < 0) return set_error(UC_EINVAL, "%s: row0 = %d must be >= 0", what, row0);
  if (bs_maps < static_cast<long>(n_max) * hs * ws)
    return set_error(UC_EINVAL, "%s: bad per-image stride %ld (>= n_max*hs*ws = %ld)", what, bs_maps, static_cast<long>(n_max) * hs * ws);
  char at[96];
  for (int b = 0; b < B; ++b) {
    snprintf(at, sizeof(at), "%s: image %d", what, b);
    if (H[b] < 1 || W[b] < 1 || !(r[b] > 0.0)) return set_error(UC_EINVAL, "%s: bad sizes", at);
  }
  if (capacity < 0) return set_error(UC_EINVAL, "%s: negative capacity", what);
  if ((reinterpret_cast<uintptr_t>(maps) | reinterpret_cast<uintptr_t>(count_dev)) % 4 || reinterpret_cast<uintptr_t>(offsets) % 8 ||
      reinterpret_cast<uintptr_t>(workspace) % 16)
    return set_error(UC_EINVAL, "%s: maps / count must be 4-byte, offsets 8-byte, workspace 16-byte aligned", what);
  const int K = B * n_max;
  MotsImages im;
  InstCover cv;
  im.n = B;
  im.k0[0] = 0;
  long diff_words = 0;
  int w_max = 0, hw32_max = 0;
  for (int b = 0; b < B; ++b) {
    snprintf(at, sizeof(at), "%s: image %d", what, b);
    const FrameResize rs = frame_resize(hs * d_rate, ws * d_rate, H[b], W[b], r[b]);
    if (rs.hm < 1 || rs.wm < 1) return set_error(UC_EINVAL, "%s: the resized mask is empty (r too large)", at);
    const int hw32 = (H[b] + 31) / 32;
    const long words = static_cast<long>(W[b]) * hw32;
    if (words > (1L << 31) / 32) return set_error(UC_EINVAL, "%s: frame too large", at);
    im.k0[b + 1] = im.k0[b] + n_max;
    im.hm[b] = H[b];
    im.wm[b] = W[b];
    im.scale[b] = rs.scale;
    im.diff0[b] = diff_words;
    cv.hv[b] = rs.hm;
    cv.wv[b] = rs.wm;
    diff_words += n_max * words;
    w_max = std::max(w_max, W[b]);
    hw32_max = std::max(hw32_max, hw32);
  }
  if (workspace_bytes < mots_workspace_bytes(K, diff_words)) return set_error(UC_EINVAL, "%s: workspace too small", what);
  MotsWs wsp = mots_ws(workspace, K, diff_words);
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  launch_pdl(inst_planes_kernel, dim3((w_max + 31) / 32, (hw32_max + 7) / 8, K), dim3(32, 8), 0, stream, maps, bs_maps, n_max, hs, ws, d_rate,
             count_dev, row0, thr, im, cv, wsp, emit);
  launch_pdl(mots_runs_kernel, K, kMotsThreads, 0, stream, static_cast<const uint8_t*>(emit), im, wsp);
  launch_pdl(mots_chars_kernel, K, kMotsThreads, 0, stream, static_cast<const uint8_t*>(emit), im, wsp, chars, capacity, offsets);
  return check_launch(what);
}
