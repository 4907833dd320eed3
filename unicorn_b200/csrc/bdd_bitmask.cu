// BDD100K MOTS "bitmask" PNG contents on the device (qdtrack core/to_bdd100k/utils.py:15-38, mask_prepare + mask_merge): every
// tracked instance's COCO RLE mask is decoded and painted in ascending score order, the last instance covering a pixel giving all four
// channels of its colour.
//   decode  one thread per string: the runs of the COCO compressed RLE (column-major, zero run first, counts after the second coded as
//           differences to the count two before) are sequential by construction.  Each string keeps its foreground runs (start pixel,
//           foreground pixels before it) in a slice of the workspace indexed by its char offset, so K strings never need more than
//           n_chars + K entries.  A malformed string paints nothing and sets its frame's status flags.
//   paint   a grid-stride loop over tiles of kBddTile foreground pixels handed out by the decode: each pixel of an instance does
//           atomicMax((rank + 1) << 16 | instance) on a column-major winner map, so consecutive pixels of a run are consecutive words
//           and the result does not depend on the order the tiles run in.
//   colour  one 32 x 32 tile per block: the column-major winner map is transposed through shared memory into the row-major RGBA frame
//           [H, W, 4] that PIL.Image.fromarray takes, 0 where no instance covers the pixel.
#include "uc_common.h"
#include "../../include/unicorn_b200.h"
#include <algorithm>
#include <climits>
#include <cstdio>

namespace uc {

constexpr int kBddMaxFrames = UC_MOTS_MAX_IMAGES;
constexpr int kBddTile = 4096;     // foreground pixels per paint task
constexpr int kBddPaintThreads = 256;
constexpr int kBddDecodeThreads = 64;
constexpr int kBddMaxInstances = 65535;  // per frame: the instance index is the low half of a winner word

// The frames of one call, passed by value: frame b owns instances [k0[b], k0[b + 1]) of the flat lists, its winner map starts at
// word map0[b] of the workspace (frames without instances have none) and its RGBA output at out[b].
struct BddFrames {
  int n;
  int k0[kBddMaxFrames + 1];
  int H[kBddMaxFrames], W[kBddMaxFrames];
  long map0[kBddMaxFrames];
  uint32_t* out[kBddMaxFrames];
};
static_assert(sizeof(BddFrames) <= 4096, "the frame descriptors must fit the kernel-parameter block");

struct BddWs {
  int* n_tasks;      // paint tasks handed out by the decode (zeroed with the maps)
  uint32_t* map;     // winner maps, column-major [W][H] per frame
  int* nfg;          // [K] foreground runs of each string (0 when malformed)
  int* start;        // [n_chars + K] first pixel of each foreground run; string j's slice starts at offsets[j] + j
  int* fgpre;        // [n_chars + K] foreground pixels before each run, then the string's total
  int2* tasks;       // {string, tile} per paint task
};
static inline long align16(long b) { return (b + 15) & ~15L; }

// Paint tasks of a frame: each instance's foreground is at most the frame, kBddTile pixels per task.
static long bdd_task_cap(int B, const int* k, const int* H, const int* W) {
  long cap = 0;
  for (int b = 0; b < B; ++b) cap += static_cast<long>(k[b]) * ((static_cast<long>(H[b]) * W[b] + kBddTile - 1) / kBddTile);
  return cap;
}
static long bdd_map_words(int B, const int* k, const int* H, const int* W, long* map0) {
  long words = 0;
  for (int b = 0; b < B; ++b) {
    if (map0) map0[b] = words;
    if (k[b] > 0) words += (static_cast<long>(H[b]) * W[b] + 3) & ~3L;
  }
  return words;
}
// [tasks counter | winner maps] (the part zeroed per call), then nfg, start, fgpre, tasks
static long bdd_ws_layout(int B, const int* k, const int* H, const int* W, long n_chars, long* map0, BddWs* ws, void* base) {
  long K = 0;
  for (int b = 0; b < B; ++b) K += k[b];
  const long zeroed = 16 + 4 * bdd_map_words(B, k, H, W, map0);
  const long runs = n_chars + K;
  const long sizes[4] = {align16(4 * K), align16(4 * runs), align16(4 * runs), align16(8 * bdd_task_cap(B, k, H, W))};
  if (ws) {
    char* p = static_cast<char*>(base);
    ws->n_tasks = reinterpret_cast<int*>(p);
    ws->map = reinterpret_cast<uint32_t*>(p + 16);
    p += align16(zeroed);
    ws->nfg = reinterpret_cast<int*>(p);
    ws->start = reinterpret_cast<int*>(p + sizes[0]);
    ws->fgpre = reinterpret_cast<int*>(p + sizes[0] + sizes[1]);
    ws->tasks = reinterpret_cast<int2*>(p + sizes[0] + sizes[1] + sizes[2]);
  }
  return align16(zeroed) + sizes[0] + sizes[1] + sizes[2] + sizes[3];
}

__device__ __forceinline__ int bdd_frame_of(const BddFrames& fr, int j) {
  int b = 0;
  while (j >= fr.k0[b + 1]) ++b;
  return b;
}

// One thread per string j: its foreground runs, its paint tasks, or its frame's status flags.
__global__ void __launch_bounds__(kBddDecodeThreads) bdd_decode_kernel(const char* __restrict__ chars, long n_chars,
                                                                      const long long* __restrict__ offsets, const int* __restrict__ ranks,
                                                                      const __grid_constant__ BddFrames fr, BddWs ws, int* __restrict__ status) {
  pdl_wait();
  pdl_launch_dependents();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= fr.k0[fr.n]) return;
  const int b = bdd_frame_of(fr, j);
  const long long hw = static_cast<long long>(fr.H[b]) * fr.W[b];
  const long long o0 = offsets[j], o1 = offsets[j + 1];
  const int rank = ranks[j];
  int flags = 0;
  if (o0 < 0 || o1 < o0 || o1 > n_chars || rank < 0 || rank >= fr.k0[b + 1] - fr.k0[b]) flags = UC_BDD_BAD_INDEX;
  int* start = ws.start + (flags ? 0 : o0 + j);
  int* fgpre = ws.fgpre + (flags ? 0 : o0 + j);
  long long pos = 0, fg = 0, c1 = 0, c2 = 0;  // c1, c2: the previous two counts
  int nfg = 0, m = 0;
  for (long long p = o0; !flags && p < o1; ++m) {
    // rleFrString (cocoapi maskApi.c): 5 data bits per char from the lowest, 0x20 = more chars follow, 0x10 in the last = negative
    long long x = 0;
    int n = 0, c = 0x20;
    while (c & 0x20) {
      if (p == o1 || n == 7) {  // the string ends inside a count, or a count longer than any frame needs
        flags = UC_BDD_BAD_CHARS;
        break;
      }
      c = chars[p++] - 48;
      if (c < 0 || c > 63) {
        flags = UC_BDD_BAD_CHARS;
        break;
      }
      x |= static_cast<long long>(c & 0x1f) << (5 * n++);
      if (!(c & 0x20) && (c & 0x10)) x |= -1LL << (5 * n);
    }
    if (flags) break;
    if (m > 2) x += c2;
    if (x < 0 || x > hw - pos) {
      flags = UC_BDD_BAD_RUNS;
      break;
    }
    if ((m & 1) && x > 0) {  // odd counts are foreground runs
      start[nfg] = static_cast<int>(pos);
      fgpre[nfg++] = static_cast<int>(fg);
      fg += x;
    }
    pos += x;
    c2 = c1;
    c1 = x;
  }
  if (!flags && pos != hw) flags = UC_BDD_BAD_RUNS;
  if (flags) {
    ws.nfg[j] = 0;
    atomicOr(status + b, flags);
    return;
  }
  fgpre[nfg] = static_cast<int>(fg);
  ws.nfg[j] = nfg;
  const int tiles = static_cast<int>((fg + kBddTile - 1) / kBddTile);
  if (tiles == 0) return;
  const int t0 = atomicAdd(ws.n_tasks, tiles);
  for (int t = 0; t < tiles; ++t) ws.tasks[t0 + t] = make_int2(j, t);
}

// Grid-stride over the paint tasks: task {j, t} paints foreground pixels [t * kBddTile, (t + 1) * kBddTile) of string j.
__global__ void __launch_bounds__(kBddPaintThreads) bdd_paint_kernel(const long long* __restrict__ offsets, const int* __restrict__ ranks,
                                                                    const __grid_constant__ BddFrames fr, BddWs ws) {
  pdl_wait();
  pdl_launch_dependents();
  const int n_tasks = *ws.n_tasks;
  for (int task = blockIdx.x; task < n_tasks; task += gridDim.x) {
    const int2 jt = ws.tasks[task];
    const int j = jt.x, b = bdd_frame_of(fr, j), nfg = ws.nfg[j];
    const long base = static_cast<long>(offsets[j]) + j;
    const int* __restrict__ start = ws.start + base;
    const int* __restrict__ fgpre = ws.fgpre + base;
    const uint32_t code = (static_cast<uint32_t>(ranks[j] + 1) << 16) | static_cast<uint32_t>(j - fr.k0[b]);
    uint32_t* map = ws.map + fr.map0[b];
    const int q1 = min(fgpre[nfg], (jt.y + 1) * kBddTile);
    int q = jt.y * kBddTile + threadIdx.x;
    if (q >= q1) continue;
    int lo = 0, hi = nfg - 1;  // the last run that starts at or before foreground pixel q
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (fgpre[mid] <= q) lo = mid;
      else hi = mid - 1;
    }
    for (int r = lo; q < q1; q += kBddPaintThreads) {
      while (fgpre[r + 1] <= q) ++r;
      atomicMax(map + start[r] + (q - fgpre[r]), code);
    }
  }
}

// One 32 x 32 pixel tile of frame blockIdx.z: winner words in column-major order, RGBA words out in row-major order.
__global__ void __launch_bounds__(256) bdd_color_kernel(const uint32_t* __restrict__ colors, const __grid_constant__ BddFrames fr, BddWs ws) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ uint32_t tile[32][33];
  const int b = blockIdx.z, H = fr.H[b], W = fr.W[b], x0 = blockIdx.x * 32, y0 = blockIdx.y * 32;
  if (x0 >= W || y0 >= H) return;
  const int k0 = fr.k0[b], tx = threadIdx.x, ty = threadIdx.y;
  const bool any = fr.k0[b + 1] > k0;
  const uint32_t* map = ws.map + fr.map0[b];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int x = x0 + ty + 8 * i, y = y0 + tx;
    uint32_t v = 0;
    if (any && x < W && y < H) v = map[static_cast<long>(x) * H + y];
    tile[ty + 8 * i][tx] = v ? colors[k0 + (v & 0xffffu)] : 0u;
  }
  __syncthreads();
  uint32_t* out = fr.out[b];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int y = y0 + ty + 8 * i, x = x0 + tx;
    if (x < W && y < H) out[static_cast<long>(y) * W + x] = tile[tx][ty + 8 * i];
  }
}

// Every host argument; false (with the error set) when one is bad.  K = the instances of all frames.
static bool bdd_check_frames(const char* what, int B, const int* k, const int* H, const int* W, long& K) {
  if (!k || !H || !W) return set_error(UC_EINVAL, "%s: null pointer", what), false;
  if (B < 1 || B > kBddMaxFrames) return set_error(UC_EINVAL, "%s: B = %d must be in 1..%d", what, B, kBddMaxFrames), false;
  K = 0;
  for (int b = 0; b < B; ++b) {
    if (H[b] < 1 || W[b] < 1 || static_cast<long>(H[b]) * W[b] > INT_MAX)
      return set_error(UC_EINVAL, "%s: frame %d: bad size %d x %d (1 <= H, W and H * W < 2^31)", what, b, H[b], W[b]), false;
    if (k[b] < 0 || k[b] > kBddMaxInstances)
      return set_error(UC_EINVAL, "%s: frame %d: k = %d must be in 0..%d", what, b, k[b], kBddMaxInstances), false;
    K += k[b];
  }
  if (bdd_task_cap(B, k, H, W) > INT_MAX) return set_error(UC_EINVAL, "%s: too many instance pixels in one call", what), false;
  return true;
}

}  // namespace uc

using namespace uc;

extern "C" long uc_bdd_bitmask_workspace_bytes(int B, const int* k, const int* H, const int* W, long n_chars) {
  long K;
  if (!bdd_check_frames("uc_bdd_bitmask_workspace_bytes", B, k, H, W, K) || n_chars < 0) return -1;
  return bdd_ws_layout(B, k, H, W, n_chars, nullptr, nullptr, nullptr);
}

extern "C" int uc_bdd_bitmask_batched(int B, const int* k, const int* H, const int* W, const long* out_offsets, const char* chars, long n_chars,
                                      const long long* offsets, const uint32_t* colors, const int* ranks, void* workspace, long workspace_bytes,
                                      uint8_t* out, long out_bytes, int* status, void* stream_v) {
  const char* what = "uc_bdd_bitmask_batched";
  long K;
  if (!bdd_check_frames(what, B, k, H, W, K)) return UC_EINVAL;
  if (!out_offsets || !offsets || !colors || !ranks || !workspace || !out || !status || (n_chars > 0 && !chars))
    return set_error(UC_EINVAL, "%s: null pointer", what);
  if (n_chars < 0 || out_bytes < 0) return set_error(UC_EINVAL, "%s: negative n_chars or out_bytes", what);
  if ((reinterpret_cast<uintptr_t>(colors) | reinterpret_cast<uintptr_t>(ranks) | reinterpret_cast<uintptr_t>(status) |
       reinterpret_cast<uintptr_t>(out)) % 4 || reinterpret_cast<uintptr_t>(offsets) % 8 || reinterpret_cast<uintptr_t>(workspace) % 16)
    return set_error(UC_EINVAL, "%s: out / colors / ranks / status must be 4-byte, offsets 8-byte, workspace 16-byte aligned", what);
  for (int b = 0; b < B; ++b) {
    const long bytes = 4L * H[b] * W[b];
    if (out_offsets[b] < 0 || out_offsets[b] % 4 || out_offsets[b] > out_bytes - bytes)
      return set_error(UC_EINVAL, "%s: frame %d: output offset %ld is not a 4-byte aligned [H, W, 4] slice of the %ld output bytes", what, b,
                       out_offsets[b], out_bytes);
    for (int c = 0; c < b; ++c)
      if (out_offsets[c] < out_offsets[b] + bytes && out_offsets[b] < out_offsets[c] + 4L * H[c] * W[c])
        return set_error(UC_EINVAL, "%s: the outputs of frames %d and %d overlap", what, c, b);
  }
  BddFrames fr;
  BddWs ws;
  fr.n = B;
  fr.k0[0] = 0;
  const long need = bdd_ws_layout(B, k, H, W, n_chars, fr.map0, &ws, workspace);
  if (workspace_bytes < need) return set_error(UC_EINVAL, "%s: workspace too small (%ld < %ld bytes)", what, workspace_bytes, need);
  int h_max = 0, w_max = 0;
  for (int b = 0; b < B; ++b) {
    fr.k0[b + 1] = fr.k0[b] + k[b];
    fr.H[b] = H[b];
    fr.W[b] = W[b];
    fr.out[b] = reinterpret_cast<uint32_t*>(out + out_offsets[b]);
    h_max = std::max(h_max, H[b]);
    w_max = std::max(w_max, W[b]);
  }
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  cudaError_t e = cudaMemsetAsync(status, 0, 4L * B, stream);
  if (e == cudaSuccess && K > 0) e = cudaMemsetAsync(workspace, 0, 16 + 4 * bdd_map_words(B, k, H, W, nullptr), stream);
  if (e != cudaSuccess) return set_error(static_cast<int>(e), "%s: %s", what, cudaGetErrorString(e));
  if (K > 0) {
    launch_pdl(bdd_decode_kernel, static_cast<int>((K + kBddDecodeThreads - 1) / kBddDecodeThreads), kBddDecodeThreads, 0, stream, chars,
               n_chars, offsets, ranks, fr, ws, status);
    const long cap = bdd_task_cap(B, k, H, W);
    launch_pdl(bdd_paint_kernel, static_cast<int>(std::min<long>(std::max<long>(cap, 1), 8L * num_sms())), kBddPaintThreads, 0, stream,
               offsets, ranks, fr, ws);
  }
  launch_pdl(bdd_color_kernel, dim3((w_max + 31) / 32, (h_max + 31) / 32, B), dim3(32, 8), 0, stream, colors, fr, ws);
  return check_launch(what);
}
