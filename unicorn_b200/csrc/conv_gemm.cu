// uc_conv2d: checks the descriptor, encodes the tensor maps and launches the conv_gemm instantiation of its epilogue variant
// (conv_gemm.cuh).
#include "conv_gemm.cuh"

namespace uc {

static int pick_block_n(int Cout, int m_tiles, int gn_gs) {
  // Heuristic default for the persistent kernel (one CTA per SM for the wide tiles): fewest waves of the widest tile
  // that does not waste more than a third of its columns.  unicorn_b200/engine.py autotunes block_n per layer on top
  // of this (plan-time timing of the candidates), so this only has to be reasonable.
  static const int cands[] = {256, 192, 128, 96, 64, 32, 16};
  const int sms = num_sms();
  int best = 0;
  double best_cost = -1.0;
  for (int bn : cands) {
    if (gn_gs > 0 && (bn % gn_gs) != 0) continue;  // GroupNorm groups must not straddle N tiles
    if (gn_gs > 0 && bn / gn_gs > kGnMaxLocal) continue;  // nor overflow the CTA's GroupNorm slots
    const int nt = (Cout + bn - 1) / bn;
    const long waste_cols = static_cast<long>(nt) * bn - Cout;
    if (waste_cols * 3 > static_cast<long>(nt) * bn && bn > 16 && gn_gs <= 0) continue;
    const long tiles = static_cast<long>(nt) * m_tiles;
    const long waves = (tiles + sms - 1) / sms;  // one persistent CTA per SM
    const double cost = static_cast<double>(waves) * (bn + 40);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = bn; }
  }
  return best;
}

}  // namespace uc

using namespace uc;

extern "C" int uc_conv2d(const UcConv2d* d, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!d || !d->x || !d->w || !d->y) return set_error(UC_EINVAL, "uc_conv2d: null pointer");
  if (d->x_dtype != UC_BF16 && d->x_dtype != UC_F16) return set_error(UC_EINVAL, "uc_conv2d: x must be bf16/f16");
  if (d->Cin % 8 || d->Cout % 8 || d->ldx % 8 || d->ldy % 8 || d->ldx < d->Cin || d->ldy < d->Cout)
    return set_error(UC_EINVAL, "uc_conv2d: Cin/Cout/ldx/ldy must be multiples of 8 (Cin=%d Cout=%d ldx=%d ldy=%d)",
                     d->Cin, d->Cout, d->ldx, d->ldy);
  if (d->stride != 1 && d->stride != 2) return set_error(UC_EINVAL, "uc_conv2d: stride must be 1 or 2");
  if (d->KH * d->KW > kMaxTaps || d->KH < 1 || d->KW < 1) return set_error(UC_EINVAL, "uc_conv2d: at most 9 taps");
  if (d->pad < 0 || d->pad >= d->KH + 1) return set_error(UC_EINVAL, "uc_conv2d: bad pad");
  if (d->res && (d->ldres % 8 || d->y_dtype == UC_F32)) return set_error(UC_EINVAL, "uc_conv2d: residual needs 16-bit y, ldres%%8==0");
  if ((reinterpret_cast<uintptr_t>(d->x) | reinterpret_cast<uintptr_t>(d->w) | reinterpret_cast<uintptr_t>(d->y) |
       reinterpret_cast<uintptr_t>(d->res)) & 15)
    return set_error(UC_EINVAL, "uc_conv2d: pointers must be 16-byte aligned");
  if (d->gn_stats && (d->gn_groups <= 0 || d->Cout % d->gn_groups))
    return set_error(UC_EINVAL, "uc_conv2d: bad GroupNorm grouping");
  if (d->act_after_res && (d->act != UC_ACT_RELU || !d->res || d->x_dtype != UC_BF16 || d->gamma || d->gn_stats || d->row_stats))
    return set_error(UC_EINVAL, "uc_conv2d: act_after_res needs act = ReLU, res and bf16 x, and excludes gamma, gn_stats and row_stats");
  if (d->row_stats && (!d->col_s || d->KH != 1 || d->KW != 1 || d->stride != 1 || d->pad != 0))
    return set_error(UC_EINVAL, "uc_conv2d: row_stats (folded LayerNorm) needs a 1x1 stride-1 conv and col_s");
  if (d->B < 1 || d->H < 1 || d->W < 1)
    return set_error(UC_EINVAL, "uc_conv2d: B, H and W must be >= 1 (B=%d H=%d W=%d)", d->B, d->H, d->W);
  // PyTorch's rule: the kernel fits in the padded map.  The numerator below is then >= 0, so C's division is the floor.
  if (d->H + 2 * d->pad < d->KH || d->W + 2 * d->pad < d->KW)
    return set_error(UC_EINVAL, "uc_conv2d: %dx%d kernel larger than the padded map (H=%d W=%d pad=%d)", d->KH, d->KW, d->H, d->W, d->pad);
  const int gn_gs = d->gn_stats ? d->Cout / d->gn_groups : 0;
  // block_n >= 1000 selects the 2-CTA cluster variant with weight multicast (1128 / 1192 / 1256)
  const bool cluster2 = d->block_n >= 1000;
  if (d->block_n) {
    const int bn = cluster2 ? d->block_n - 1000 : d->block_n;
    if (cluster2 && bn != 128 && bn != 192 && bn != 256)
      return set_error(UC_EINVAL, "uc_conv2d: the cluster variant exists for block_n 128/192/256 only");
    if (bn != 16 && bn != 32 && bn != 64 && bn != 96 && bn != 128 && bn != 192 && bn != 256)
      return set_error(UC_EINVAL, "uc_conv2d: unsupported block_n %d", d->block_n);
    if (gn_gs && bn % gn_gs) return set_error(UC_EINVAL, "uc_conv2d: N tile %d incompatible with GroupNorm group size %d", bn, gn_gs);
    if (gn_gs && bn / gn_gs > kGnMaxLocal)
      return set_error(UC_EINVAL, "uc_conv2d: N tile %d holds %d GroupNorm groups, more than the %d a CTA accumulates", bn, bn / gn_gs,
                       kGnMaxLocal);
  }

  const int s = d->stride;
  const int Ho = (d->H + 2 * d->pad - d->KH) / s + 1;
  const int Wo = (d->W + 2 * d->pad - d->KW) / s + 1;

  ConvKernelParams p;
  memset(&p, 0, sizeof(p));
  const CUtensorMapDataType dt = d->x_dtype == UC_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const bool flat = (d->KH == 1 && d->KW == 1 && s == 1 && d->pad == 0);
  int B = d->B, Hm = d->H, Wm = d->W;  // map geometry
  // a flat conv is one row of H*W pixels per image; the batch stays the 4th map dimension, so no tile spans two images and each
  // tile's GroupNorm sums go to its own image's slot
  if (flat) { Wm = d->H * d->W; Hm = 1; }
  p.Wo = flat ? Wm : Wo;
  p.Ho = flat ? 1 : Ho;
  p.B = B;
  // tile shape minimising the number of 128-pixel tiles
  {
    int best_tw = 128, best_th = 1;
    long best = -1;
    for (int tw = 128; tw >= 8; tw >>= 1) {
      const int th = 128 / tw;
      const long n = static_cast<long>((p.Wo + tw - 1) / tw) * ((p.Ho + th - 1) / th);
      if (best < 0 || n < best) { best = n; best_tw = tw; best_th = th; }
    }
    p.tile_w = best_tw; p.tile_h = best_th;
  }
  p.tiles_w = (p.Wo + p.tile_w - 1) / p.tile_w;
  p.tiles_h = (p.Ho + p.tile_h - 1) / p.tile_h;
  const int m_tiles = p.tiles_w * p.tiles_h * B;

  // A stride phase of a map one pixel high or wide has no pixels (phase 1 of W = 1 at stride 2): its tensor map is not encoded, and
  // the taps that fall on it read only zero padding, so they are left out.  t.tap still indexes the packed weights.
  auto phase_empty = [&](int ph, int pw) { return (Wm - pw + s - 1) / s <= 0 || (Hm - ph + s - 1) / s <= 0; };
  int nt = 0;
  for (int kh = 0; kh < d->KH; ++kh) {
    for (int kw = 0; kw < d->KW; ++kw) {
      const int offh = kh - d->pad, offw = kw - d->pad;
      const int ph = ((offh % s) + s) % s, pw = ((offw % s) + s) % s;
      if (phase_empty(ph, pw)) continue;
      ConvTap t;
      t.map = static_cast<int16_t>(ph * s + pw);
      t.dh = static_cast<int16_t>((offh - ph) / s);
      t.dw = static_cast<int16_t>((offw - pw) / s);
      t.tap = static_cast<int16_t>(kh * d->KW + kw);
      p.taps[nt++] = t;
    }
  }
  if (nt == 0)
    return set_error(UC_EINVAL, "uc_conv2d: every tap of this %dx%d stride-2 conv reads only zero padding (H=%d W=%d pad=%d)", d->KH,
                     d->KW, d->H, d->W, d->pad);
  p.ntaps = nt;
  p.kchunks = (d->Cin + kBlockK - 1) / kBlockK;
  const int bn = cluster2 ? d->block_n - 1000 : d->block_n ? d->block_n : pick_block_n(d->Cout, m_tiles, gn_gs);
  if (bn == 0) return set_error(UC_EINVAL, "uc_conv2d: no N tile compatible with GroupNorm group size %d", gn_gs);

  int rc = ensure_driver();
  if (rc) return rc;
  // activation maps: one per stride phase
  const size_t es = 2;
  for (int ph = 0; ph < s; ++ph) {
    for (int pw = 0; pw < s; ++pw) {
      const int Wp = (Wm - pw + s - 1) / s, Hp = (Hm - ph + s - 1) / s;
      if (phase_empty(ph, pw)) continue;
      const uint8_t* base = reinterpret_cast<const uint8_t*>(d->x) + (static_cast<size_t>(ph) * Wm + pw) * d->ldx * es;
      uint64_t dims[4] = {static_cast<uint64_t>(d->Cin), static_cast<uint64_t>(Wp), static_cast<uint64_t>(Hp), static_cast<uint64_t>(B)};
      uint64_t strides[3] = {static_cast<uint64_t>(s) * d->ldx * es, static_cast<uint64_t>(s) * Wm * d->ldx * es,
                             static_cast<uint64_t>(Hm) * Wm * d->ldx * es};
      uint32_t box[4] = {static_cast<uint32_t>(kBlockK), static_cast<uint32_t>(p.tile_w), static_cast<uint32_t>(p.tile_h), 1};
      rc = encode_tmap(&p.tmA[ph * s + pw], dt, 4, base, dims, strides, box);
      if (rc) return rc;
    }
  }

  const int ktaps = d->KH * d->KW;  // taps of the packed weights
  {
    uint64_t dims[3] = {static_cast<uint64_t>(d->Cin), static_cast<uint64_t>(ktaps), static_cast<uint64_t>(d->Cout)};
    uint64_t strides[2] = {static_cast<uint64_t>(d->Cin) * es, static_cast<uint64_t>(ktaps) * d->Cin * es};
    uint32_t box[3] = {static_cast<uint32_t>(kBlockK), 1, static_cast<uint32_t>(bn)};
    rc = encode_tmap(&p.tmB, dt, 3, d->w, dims, strides, box);
    if (rc) return rc;
  }
  p.Cout = d->Cout;
  p.bias = d->bias; p.gamma = d->gamma; p.res = d->res; p.ldres = d->ldres;
  p.y = d->y; p.ldy = d->ldy; p.y_dtype = d->y_dtype; p.act = d->act_after_res ? UC_ACT_NONE : d->act; p.relu_res = d->act_after_res;
  p.row_stats = static_cast<const long long*>(d->row_stats); p.col_s = d->col_s; p.row_inv = 1.f / (kGnFixedScale * static_cast<float>(d->Cin)); p.row_eps = d->row_eps;
  p.gn_stats = static_cast<long long*>(d->gn_stats); p.gn_groups = d->gn_groups;
  p.gn_gs = d->gn_stats ? gn_gs : 1 << 30;
  p.n_tiles = (d->Cout + bn - 1) / bn;
  p.m_tiles = m_tiles;
  if (d->y_dtype != UC_F32) {  // 16-bit y (and the residual, same dtype and geometry) moves by TMA through the staging tile
    const int slab = conv_slab(bn);
    const CUtensorMapSwizzle swz = slab == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : slab == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
    const CUtensorMapDataType ydt = d->y_dtype == UC_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    uint64_t dims[4] = {static_cast<uint64_t>(d->Cout), static_cast<uint64_t>(p.Wo), static_cast<uint64_t>(p.Ho), static_cast<uint64_t>(B)};
    uint32_t box[4] = {static_cast<uint32_t>(slab), static_cast<uint32_t>(p.tile_w), static_cast<uint32_t>(p.tile_h), 1};
    for (int r = 0; r < (d->res ? 2 : 1); ++r) {
      const uint64_t ld = static_cast<uint64_t>(r ? d->ldres : d->ldy) * es;
      uint64_t strides[3] = {ld, ld * p.Wo, ld * p.Wo * p.Ho};
      rc = encode_tmap(r ? &p.tmR : &p.tmY, ydt, 4, r ? d->res : d->y, dims, strides, box, swz);
      if (rc) return rc;
    }
  }
  const bool f16 = d->x_dtype == UC_F16;
  if (cluster2) {
    uint64_t dims[3] = {static_cast<uint64_t>(d->Cin), static_cast<uint64_t>(ktaps), static_cast<uint64_t>(d->Cout)};
    uint64_t strides[2] = {static_cast<uint64_t>(d->Cin) * es, static_cast<uint64_t>(ktaps) * d->Cin * es};
    uint32_t box[3] = {static_cast<uint32_t>(kBlockK), 1, static_cast<uint32_t>(bn / 2)};
    rc = encode_tmap(&p.tmBh, dt, 3, d->w, dims, strides, box);
    if (rc) return rc;
  }
  // the fixed epilogue variants (bf16 operands) cover every combination the engine issues; anything else runs kEpiAny
  if (f16) return conv_launch<kEpiAny, true>(p, bn, cluster2, stream);
  const bool bf16y = d->y_dtype == UC_BF16, plain = !d->gamma && !d->res && !d->gn_stats && !d->row_stats;
  int epi = kEpiAny;
  if (d->act_after_res) epi = bf16y ? kEpiReluRes : kEpiAny;
  else if (d->res) epi = bf16y && d->act == UC_ACT_NONE && !d->gn_stats && !d->row_stats ? kEpiRes : kEpiAny;
  else if (d->gn_stats) epi = bf16y && d->act == UC_ACT_NONE && !d->gamma && !d->row_stats ? kEpiGn : kEpiAny;
  else if (d->row_stats) epi = bf16y && d->act == UC_ACT_GELU && !d->gamma ? kEpiGeluLn : kEpiAny;
  else if (!plain) epi = kEpiAny;
  else if (d->y_dtype == UC_F32) epi = d->act == UC_ACT_NONE ? kEpiF32 : kEpiAny;
  else if (d->y_dtype == UC_F16) epi = d->act == UC_ACT_NONE ? kEpiBiasF16 : kEpiAny;
  else if (d->act == UC_ACT_NONE) epi = kEpiBias;
  else if (d->act == UC_ACT_RELU) epi = kEpiRelu;
  else if (d->act == UC_ACT_GELU) epi = kEpiGelu;
  switch (epi) {
    case kEpiBias: return conv_launch<kEpiBias, false>(p, bn, cluster2, stream);
    case kEpiBiasF16: return conv_launch<kEpiBiasF16, false>(p, bn, cluster2, stream);
    case kEpiF32: return conv_launch<kEpiF32, false>(p, bn, cluster2, stream);
    case kEpiRelu: return conv_launch<kEpiRelu, false>(p, bn, cluster2, stream);
    case kEpiGelu: return conv_launch<kEpiGelu, false>(p, bn, cluster2, stream);
    case kEpiGeluLn: return conv_launch<kEpiGeluLn, false>(p, bn, cluster2, stream);
    case kEpiRes: return conv_launch<kEpiRes, false>(p, bn, cluster2, stream);
    case kEpiReluRes: return conv_launch<kEpiReluRes, false>(p, bn, cluster2, stream);
    case kEpiGn: return conv_launch<kEpiGn, false>(p, bn, cluster2, stream);
    default: return conv_launch<kEpiAny, false>(p, bn, cluster2, stream);
  }
}
