// h264_inter.cu — P pictures: one warp per macroblock, P_L0_16x16 (ITU-T H.264 8.4).
//
//  1. the 16x16 source block and a 48x48 window of the previous reconstruction (L2-resident: a 4K
//     NV12 frame is 12.4 MB against 50 MB of L2) are staged in shared memory;
//  2. exhaustive full-sample search, dx in [-16,15] (one candidate column per LANE), dy in [-16,16]:
//     every window row is byte-aligned once per lane with funnel shifts and then feeds the 16 (row, dy)
//     pairs it belongs to — 33 SAD accumulators live in registers, VABSDIFF4.U8.ACC does 4 pixels per
//     instruction; cost = SAD + lambda*(bits(mvx)+bits(mvy)); the arg-min is a single warp-wide
//     REDUX.MIN over (cost << 11 | candidate index);
//  3. quarter-sample refinement: the half-sample planes (6-tap) around the winner are built in shared memory, every
//     fractional position is one plane row or the byte-wise rounded average of two (Table 8-12 as data, __vavgu4), 8 half-
//     then 8 quarter-sample candidates are scored with VABSDIFF4 on whole rows (lane = candidate half x row);
//  4. prediction (luma from the planes, chroma 1/8-sample bilinear), residual transform/quantisation and
//     reconstruction with one lane per 4x4 block (h264_common.cuh).
// Three passes per picture (DESIGN.md §5.3).  k_inter_lean takes every macroblock in raster order and finishes the ones that leave
// through the zero vector or an unrefined temporal-predictor hit — most of a desktop picture — without the search's registers and
// shared memory; it queues the rest.  k_inter_search then runs twice: over the queued anchors, then over everything else queued,
// which reads the anchors' vectors.  Both kernels take a macroblock's early exits through the same functions (start_mb,
// temporal_predictor, stage_pred_window, test_candidate) on inputs that nothing writes during the analysis of a picture, so a queued
// macroblock's tests decide in k_inter_search as they did in k_inter_lean.  Apart from the anchors' vectors, there is no dependency
// between macroblocks of a P picture: motion-vector prediction and the P_Skip decision only matter for entropy coding and are
// resolved in h264_entropy.cu.
// Encoder decisions: DESIGN.md §5.3; CPU restatement: oracle/h264_ref.c encode_inter_mb().
#include "h264_common.cuh"
#include "h264_kernels.h"

namespace b2v {

constexpr int WIN_ROWS = 48, WIN_WORDS = 12;
constexpr int PW_ROWS = 24, PW_WORDS = 8;      // the part of the window around a temporal predictor (k_inter_lean)
constexpr int WARPS_PER_BLOCK = 4;

struct alignas(16) InterSm {      // one per warp; the 16-byte size padding keeps t's uint4 accesses aligned for every array element
  MbTile t;
  uint32_t win[WIN_ROWS][WIN_WORDS];
  // quarter-sample refinement (8.4.2.2.1): planes around the best full-sample position, sample (X,Y) relative to it
  alignas(4) int16_t b1[22][18];   // unrounded horizontal 6-tap, b1[Y+3][X+1], Y in [-3,18], X in [-1,15]
  alignas(4) uint8_t bq[18][24];   // b = clip((b1+16)>>5),          bq[Y+1][X+1], Y in [-1,16], X in [-1,15]
  alignas(4) uint8_t hq[17][24];   // vertical half sample,          hq[Y+1][X+1], Y in [-1,15], X in [-1,16]
  alignas(4) uint8_t jq[17][24];   // centre half sample,            jq[Y+1][X+1], Y,X in [-1,15]
};
struct alignas(16) LeanSm {       // one per warp of k_inter_lean
  MbTile t;
  uint32_t pw[PW_ROWS][PW_WORDS];
};
// rows [r0, ...) x words [w0, w0 + stride) of the 48 x 12-word window, stored densely: the whole window or the k_inter_lean part
struct WinView {
  uint32_t* p;
  int stride, r0, w0;
  __device__ __forceinline__ uint32_t* at(int r, int w) const { return p + (r - r0) * stride + (w - w0); }
};

constexpr int ME_PRED_SAD_FACTOR = 4;      // temporal predictor accepted up to 4x the early-termination threshold (and only as a strict local minimum)
constexpr int ME_FRAC_PENALTY_BITS = 4;   // fractional vectors pay 4 extra bits in the refinement cost
constexpr int ME_REFINE_MAX_SAD = 8192;   // no sub-sample refinement of a full-sample match this bad
constexpr int ME_NEWCONTENT_DY = 2;       // vertical range of the reduced search on new content

// ---- B2V_FLAG_WIDE_MOTION (DESIGN.md §5.3; oracle/h264_wide_ref.c coarse_search, encode_inter_mb_wide) ----
// A full-sample vector is usable when each component lies in [-255, 255]: with a quarter-sample refinement (+-3/4) every coded
// component then lies in [-1024, 1023] quarter samples, the range the SPS asserts (VUI log2_max_mv_length_* = 10), inside Table A-1's
// MaxVmvR of every level it writes.
constexpr int MV_MAX_FULL = 255;
constexpr int WM_DX = 32, WM_DY = 64;      // coarse search: dx in [-32, 31], dy in [-64, 63] decimated samples (x4 luma samples)
constexpr int COARSE_NONE = 0x7fffffff;
constexpr int WM_MVD_BITS = 48;            // header budget of a P macroblock in a wide-motion picture: 48 more bits for two mvd of up to +-2046
__device__ __forceinline__ bool mv_ok(int kx, int ky) { return kx >= -MV_MAX_FULL && kx <= MV_MAX_FULL && ky >= -MV_MAX_FULL && ky <= MV_MAX_FULL; }

// Table 8-12 as data: every fractional position is one plane sample or the rounded average of two.
// entry = p1 | dx1<<2 | dy1<<3 | p2<<4 | dx2<<7 | dy2<<8, planes 0 G (full sample), 1 b, 2 h, 3 j, p2 = 4: none
__device__ const uint16_t subpel_tab[16] = {
  /* fy=0 */ 0 | (4 << 4),            0 | (1 << 4),             1 | (4 << 4),            0 | (1 << 2) | (1 << 4),
  /* fy=1 */ 0 | (2 << 4),            1 | (2 << 4),             1 | (3 << 4),            1 | (2 << 4) | (1 << 7),
  /* fy=2 */ 2 | (4 << 4),            2 | (3 << 4),             3 | (4 << 4),            3 | (2 << 4) | (1 << 7),
  /* fy=3 */ 0 | (1 << 3) | (2 << 4), 2 | (1 << 4) | (1 << 8),  3 | (1 << 4) | (1 << 8), 2 | (1 << 2) | (1 << 4) | (1 << 8),
};

__device__ __forceinline__ int se_bits_dev(int v) {
  const unsigned c = (v > 0 ? 2u * (unsigned)v - 1u : (unsigned)(-2 * v)) + 1u;
  return 2 * (31 - __clz(c)) + 1;
}
// 16 consecutive bytes starting at an arbitrarily aligned shared-memory address -> 4 words
__device__ __forceinline__ void load_row16(const uint8_t* p, uint32_t out[4]) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  const int sh = (a & 3) * 8;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(p - (a & 3));
  const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = w[4];
  out[0] = __funnelshift_r(w0, w1, sh); out[1] = __funnelshift_r(w1, w2, sh); out[2] = __funnelshift_r(w2, w3, sh); out[3] = __funnelshift_r(w3, w4, sh);
}
__device__ __forceinline__ const uint8_t* plane_ptr(const InterSm& sm, int plane, int ox, int oy, int X, int Y) {
  return plane == 0 ? reinterpret_cast<const uint8_t*>(&sm.win[oy + Y][0]) + ox + X
       : plane == 1 ? &sm.bq[Y + 1][X + 1] : plane == 2 ? &sm.hq[Y + 1][X + 1] : &sm.jq[Y + 1][X + 1];
}
// predicted luma row `row` (16 samples) for the quarter-sample offset (qx,qy) in [-3,3] from the full-sample position (ox,oy)
__device__ __forceinline__ void subpel_row(const InterSm& sm, int ox, int oy, int qx, int qy, int row, uint32_t out[4]) {
  const int xi = qx >> 2, yi = qy >> 2;
  const uint32_t e = subpel_tab[(qy & 3) * 4 + (qx & 3)];
  load_row16(plane_ptr(sm, e & 3, ox, oy, xi + ((e >> 2) & 1), row + yi + ((e >> 3) & 1)), out);
  const int p2 = (e >> 4) & 7;
  if (p2 < 4) {
    uint32_t o2[4];
    load_row16(plane_ptr(sm, p2, ox, oy, xi + ((e >> 7) & 1), row + yi + ((e >> 8) & 1)), o2);
#pragma unroll
    for (int k = 0; k < 4; k++) out[k] = __vavgu4(out[k], o2[k]);      // (a + b + 1) >> 1 per byte
  }
}

__device__ __forceinline__ uint32_t sad4acc(uint32_t a, uint32_t b, uint32_t c) {   // VABSDIFF4.U8.ACC with a live accumulator
  uint32_t d; asm("vabsdiff4.u32.u32.u32.add %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d;
}

__host__ __device__ constexpr int se_bits_c(int v) {
  unsigned c = (v > 0 ? 2u * (unsigned)v - 1u : (unsigned)(-2 * v)) + 1u;
  int len = 0;
  while ((c >> len) > 1) len++;
  return 2 * len + 1;
}

// Full-sample search over dx in [-16,15] (one candidate column per lane) and dy in [-DYR,DYR]: every window row is byte-aligned once
// per lane with funnel shifts and feeds the (row, dy) pairs it belongs to; 2*DYR+1 SAD accumulators live in registers.  Returns the
// warp-wide minimum of cost << 11 | candidate index.  DYR = 16 is the exhaustive search, a small DYR the reduced one for new content.
// WIDE: the window is centred on the full-sample vector (ox, oy); costs are those of the real vectors and candidates outside
// MV_MAX_FULL are skipped.
template <int DYR, bool WIDE = false>
__device__ __forceinline__ uint32_t search_rows(const InterSm& sm, int lane, int lambda, int ox = 0, int oy = 0) {
  const MbTile& t = sm.t;
  uint32_t c[16][4];
#pragma unroll
  for (int r = 0; r < 16; r++) {
    const uint4 v = *reinterpret_cast<const uint4*>(&t.cur_y[r][0]);
    c[r][0] = v.x; c[r][1] = v.y; c[r][2] = v.z; c[r][3] = v.w;
  }
  constexpr int N = 2 * DYR + 1, Y0 = 16 - DYR;
  uint32_t acc[N];
#pragma unroll
  for (int i = 0; i < N; i++) acc[i] = 0;
  const int wi = lane >> 2, sh = (lane & 3) * 8;
#pragma unroll
  for (int y = Y0; y < Y0 + N + 15; y++) {
    const uint32_t* wr = sm.win[y] + wi;
    const uint32_t w0 = wr[0], w1 = wr[1], w2 = wr[2], w3 = wr[3], w4 = wr[4];
    const uint32_t a0 = __funnelshift_r(w0, w1, sh), a1 = __funnelshift_r(w1, w2, sh), a2 = __funnelshift_r(w2, w3, sh), a3 = __funnelshift_r(w3, w4, sh);
#pragma unroll
    for (int r = 0; r < 16; r++) {
      const int k = y - r - Y0;
      if (k >= 0 && k < N)
        acc[k] = sad4acc(c[r][0], a0, sad4acc(c[r][1], a1, sad4acc(c[r][2], a2, sad4acc(c[r][3], a3, acc[k]))));
    }
  }
  const int bits_x = WIDE ? se_bits_dev(4 * (ox + lane - 16)) : se_bits_c(4 * (lane - 16));
  uint32_t best = 0xffffffffu;
#pragma unroll
  for (int k = 0; k < N; k++) {
    const int dyi = k + Y0;                     // dy + 16
    const uint32_t cost = acc[k] + (uint32_t)(lambda * (bits_x + (WIDE ? se_bits_dev(4 * (oy + dyi - 16)) : se_bits_c(4 * (dyi - 16)))));
    if (!WIDE || mv_ok(ox + lane - 16, oy + dyi - 16)) best = min(best, (cost << 11) | (uint32_t)(dyi * 32 + lane));
  }
  return __reduce_min_sync(FULL, best);
}

// A macroblock's place: its band's first row and the anchor of its 4x4 group — one per group, at offset (1,1), groups counted inside
// each band (oracle/h264_ref.c anchor_of()).  An anchor's vector is the first candidate of the other macroblocks of its group whose
// temporal predictor failed.  `inside`: the window's 48 columns lie inside the picture, so it needs no per-sample clamping.
struct MbPos {
  int mb, mbx, mby, band_r0, ax, ay;
  bool anchor, inside;
};
__device__ __forceinline__ MbPos mb_pos(const FrameCtx& f, int mb) {
  MbPos p;
  p.mb = mb; p.mby = mb / f.mbw; p.mbx = mb - p.mby * f.mbw;
  p.band_r0 = p.mby / f.band_rows * f.band_rows;
  p.ax = min(4 * (p.mbx >> 2) + 1, f.mbw - 1);
  p.ay = p.band_r0 + min(4 * ((p.mby - p.band_r0) >> 2) + 1, min(f.mbh - p.band_r0, f.band_rows) - 1);
  p.anchor = p.ax == p.mbx && p.ay == p.mby;
  p.inside = p.mbx >= 1 && p.mbx * 16 + 32 <= f.cw;
  return p;
}

// With B2V_FLAG_DROPPABLE the previous picture's vector spans f.prev_ref_dist pictures and this picture's reference lies f.ref_dist
// pictures back (1 or 2 each), so as a temporal predictor the vector is scaled by ref_dist / prev_ref_dist: doubled exactly, or halved
// rounding half away from zero, v -> sign(v) * ((|v| + 1) >> 1) (oracle/h264_layers_ref.c scale_mv).  Both distances are 1 without the flag;
// the kernels are instantiated with SCALE = false for pictures whose two distances are equal, which then run the code of a build
// without layers.
__device__ __forceinline__ int scale_mv(int v, int num, int den) {
  const int s = v >> 31, h = ((((v ^ s) - s) + 1) >> 1 ^ s) - s;
  return num == den ? v : num > den ? 2 * v : h;
}

// The start of a macroblock in both passes: one batch of independent global loads — the source block, staged into the tile, the
// co-located luma block z and, speculatively (otherwise they cost a dependent-load latency later), the co-located chroma reference
// (the chroma prediction of a zero vector) and the previous picture's record (temporal predictor; its vector scaled to this
// picture's reference distance) — and SAD(0,0) from the source and z as loaded.  The tile is read by other lanes after a __syncwarp.
struct MbStart { uint32_t uv_coloc; uint2 z; MbInfo prev; int sad0; };
template <bool SCALE>
__device__ __forceinline__ MbStart start_mb(const FrameCtx& f, MbTile& t, int lane, const MbPos& p) {
  const size_t ysz = (size_t)f.cw * f.ch;
  const int x0 = p.mbx * 16, r8 = lane >> 1, c8 = (lane & 1) * 8;
  MbStart s;
  s.uv_coloc = __ldg(reinterpret_cast<const uint32_t*>(f.ref + ysz + (size_t)(p.mby * 8 + (lane >> 2)) * f.cw + x0 + (lane & 3) * 4));
  s.z = __ldg(reinterpret_cast<const uint2*>(f.ref + (size_t)(p.mby * 16 + r8) * f.cw + x0 + c8));
  s.prev = f.mbinfo_prev[p.mb];
  if (SCALE) { s.prev.mvx = (int16_t)scale_mv(s.prev.mvx, f.ref_dist, f.prev_ref_dist); s.prev.mvy = (int16_t)scale_mv(s.prev.mvy, f.ref_dist, f.prev_ref_dist); }
  const uint2 c = stage_source(f, t, lane, x0, p.mby, ysz);
  s.sad0 = __reduce_add_sync(FULL, (int)sad4acc(c.x, s.z.x, sad4acc(c.y, s.z.y, 0u)));
  return s;
}

// ---- temporal-predictor early termination (DESIGN.md §5.3; oracle/h264_ref.c encode_inter_mb / try_candidate) ----
// A vector (quarter samples) as a full-sample candidate (kx,ky); true when the candidate's 3x3 test lies inside the window.
__device__ __forceinline__ bool full_sample_candidate(int mvx, int mvy, int& kx, int& ky) {
  kx = (mvx + 2) >> 2; ky = (mvy + 2) >> 2;
  return kx >= -15 && kx <= 14 && ky >= -15 && ky <= 15;
}
// The temporal predictor: the vector this macroblock had in the previous picture, rounded to full samples (scrolling and panning
// content repeats it; the zero vector counts: static content whose co-located SAD sits just above the early-termination threshold
// would otherwise search only to find (0,0) again), and the 24 rows x 8 words of the window from (ra, wa) on that its test, a refinement
// around it and its prediction touch: rows [13+cdy, 36+cdy] and bytes [13+cdx, 34+cdx] cover the 3x3 test (rows 15+cdy..32+cdy), the
// 6-tap support (-3..+18) and the prediction, clamped so that they stay inside the window.  `prev`: as start_mb scaled it.
// WIDE: a predictor outside the co-located window's test range but within MV_MAX_FULL is tested in the window centred on (wx, wy) =
// (its x rounded down to a multiple of 4, so that the window's rows stay word-aligned, its y); (cdx, cdy) is relative to that centre.
struct TemporalPred { int cdx, cdy, ra, wa; bool try_pred; int wx, wy; };
template <bool WIDE>
__device__ __forceinline__ TemporalPred temporal_predictor(const MbInfo& prev) {
  TemporalPred tp;
  tp.wx = 0; tp.wy = 0;
  bool in = full_sample_candidate(prev.mvx, prev.mvy, tp.cdx, tp.cdy);
  if (WIDE && !in && mv_ok(tp.cdx, tp.cdy)) { tp.wx = tp.cdx & ~3; tp.wy = tp.cdy; tp.cdx -= tp.wx; tp.cdy = 0; in = true; }
  tp.try_pred = in && prev.type == MB_P16;
  tp.ra = min(max(13 + tp.cdy, 0), WIN_ROWS - PW_ROWS); tp.wa = min(max((13 + tp.cdx) >> 2, 0), WIN_WORDS - PW_WORDS);
  return tp;
}
// the 48 columns of the window centred on (wx, *) lie inside the picture (MbPos::inside for wx = 0)
__device__ __forceinline__ bool window_inside(const FrameCtx& f, const MbPos& p, int wx) { return p.mbx * 16 - 16 + wx >= 0 && p.mbx * 16 + 32 + wx <= f.cw; }
// Those 24 rows x 8 words (a macroblock whose window lies inside the picture) into `dst`: the whole window or k_inter_lean's dense
// copy of that part, so that both passes test the predictor on the same words at the same window coordinates.
__device__ __forceinline__ void stage_pred_window(const FrameCtx& f, const WinView& dst, int lane, const MbPos& p, int ylo, int yhi, const TemporalPred& tp) {
  const uint32_t* base = reinterpret_cast<const uint32_t*>(f.ref + p.mbx * 16 - 16 + tp.wx);
  uint32_t v[6];
#pragma unroll
  for (int k = 0; k < 6; k++) {
    const int idx = lane + 32 * k;
    v[k] = __ldg(base + (size_t)clip3i(ylo, yhi, p.mby * 16 - 16 + tp.wy + tp.ra + (idx >> 3)) * (f.cw >> 2) + tp.wa + (idx & 7));
  }
#pragma unroll
  for (int k = 0; k < 6; k++) {
    const int idx = lane + 32 * k;
    *dst.at(tp.ra + (idx >> 3), tp.wa + (idx & 7)) = v[k];
  }
  __syncwarp();
}

// the SAD of a candidate key (cost << 11 | candidate index) whose vector is (mvx, mvy), quarter samples
__device__ __forceinline__ int key_sad(uint32_t key, int lambda, int mvx, int mvy) { return (int)(key >> 11) - lambda * (se_bits_dev(mvx) + se_bits_dev(mvy)); }

// Candidate (kx,ky), full samples, window staged around it: true (and `best` = its key) when its SAD is within 4x the noise
// threshold AND it is a strict local minimum of the cost over its 8 full-sample neighbours AND it costs no more than the zero vector.
// (kx, ky) relative to the window's centre (ox, oy); costs are those of the real vector.
__device__ __forceinline__ bool test_candidate(const WinView& w, const MbTile& t, int lane, int kx, int ky, int lambda, int sad0, uint32_t& best, int ox = 0, int oy = 0) {
  const int r8 = lane >> 1, c8 = (lane & 1) * 8;
  const uint32_t c0 = *reinterpret_cast<const uint32_t*>(&t.cur_y[r8][c8]), c1 = *reinterpret_cast<const uint32_t*>(&t.cur_y[r8][c8 + 4]);
  uint32_t kc = 0, kmin = 0xffffffffu;
#pragma unroll
  for (int j = -1; j <= 1; j++) {
#pragma unroll
    for (int i = -1; i <= 1; i++) {
      const int bx = 16 + kx + i + c8;
      const uint32_t* wr = w.at(16 + ky + j + r8, bx >> 2);
      const int sh = (bx & 3) * 8;
      const uint32_t a0 = __funnelshift_r(wr[0], wr[1], sh), a1 = __funnelshift_r(wr[1], wr[2], sh);
      const int sad = __reduce_add_sync(FULL, (int)sad4acc(c0, a0, sad4acc(c1, a1, 0u)));
      const uint32_t cost = (uint32_t)(sad + lambda * (se_bits_dev(4 * (ox + kx + i)) + se_bits_dev(4 * (oy + ky + j))));
      const uint32_t key = (cost << 11) | (uint32_t)((ky + j + 16) * 32 + (kx + i + 16));
      if (i == 0 && j == 0) kc = key; else kmin = min(kmin, key);
    }
  }
  const uint32_t key0 = ((uint32_t)(sad0 + 2 * lambda) << 11) | (uint32_t)(16 * 32 + 16);   // ... and it must not cost more than the zero vector
  if (key_sad(kc, lambda, 4 * (ox + kx), 4 * (oy + ky)) <= ME_PRED_SAD_FACTOR * ME_EARLY_SAD_PER_LAMBDA * lambda && kc < kmin && kc <= key0) { best = kc; return true; }
  return false;
}

// full-sample luma prediction at window position (dxi, dyi) into the tile: 8 samples of window row dyi + r8 per lane
__device__ __forceinline__ void full_sample_pred(const WinView& w, MbTile& t, int lane, int dxi, int dyi) {
  const int r8 = lane >> 1, c8 = (lane & 1) * 8;
  const int bo = dxi + c8;
  const uint32_t* wr = w.at(dyi + r8, bo >> 2);
  const int sh = (bo & 3) * 8;
  *reinterpret_cast<uint32_t*>(&t.pred_y[r8][c8]) = __funnelshift_r(wr[0], wr[1], sh);
  *reinterpret_cast<uint32_t*>(&t.pred_y[r8][c8 + 4]) = __funnelshift_r(wr[1], wr[2], sh);
}

// an anchor's vector for the rest of its group: one 8-byte store, tag and vector together.  WIDE: 12 bits per component,
// (mvx & 0xfff) << 20 | new-content flag << 16 | mvy & 0xfff
template <bool WIDE>
__device__ __forceinline__ void publish_anchor(const FrameCtx& f, int mb, int sad_int, int mvx, int mvy) {
  if (WIDE) f.me_pub[mb] = ((unsigned long long)((uint32_t)f.pic + 1u) << 32) | (sad_int >= ME_REFINE_MAX_SAD ? 0x10000u : 0u) | ((uint32_t)(mvx & 0xfff) << 20) | (uint32_t)(mvy & 0xfff);
  else f.me_pub[mb] = ((unsigned long long)((uint32_t)f.pic + 1u) << 32) | (sad_int >= ME_REFINE_MAX_SAD ? 0x10000u : 0u) | (uint32_t)((mvx & 0xff) << 8) | (uint32_t)(mvy & 0xff);
}

// chroma prediction, residual, reconstruction and the macroblock's record; the luma prediction is already in t.pred_y.
// uv_coloc: this lane's word of the co-located chroma reference.  ltr (B2V_FLAG_LONG_TERM_REF): the vector (LTR_MV, LTR_MV), which
// no macroblock can have, stands for refIdx 1, the zero vector into the long-term picture.  The I_PCM header budget holds for it
// unchanged: its mvd is -mvp, no longer than the mvd of a vector of the same range, and ref_idx_l0 (te(v), one bit, in every
// P_L0_16x16 macroblock of a picture with two references) fits: 1 (mb_type) + 2 x 17 (mvd of +-134 quarter samples) + 11
// (coded_block_pattern) + 1 (mb_qp_delta) = 47 bits without it, 48 with it; with wide-range motion 2 x 23 bits of mvd, 60 of
// 48 + WM_MVD_BITS.
constexpr int LTR_MV = -32768;
constexpr uint32_t LTR_MV_WORD = 0x80008000u;
template <bool WIDE>
__device__ __forceinline__ void code_p_mb(const FrameCtx& f, MbTile& t, int lane, int mb, int qp, uint32_t mv, bool ltr, size_t ysz);
// SIDE: what the picture-level decisions after the analysis need of the macroblock.
//  * SIDE_COST (B2V_FLAG_SCENE_CUT): its cost_inter into f.scut_cost, the value the exits and the search compare: the luma SAD of the prediction plus
//    lambda x (bits of the vector's components, + ME_FRAC_PENALTY_BITS for a fractional vector); the zero vector's for refIdx 1.
//    0 when the SAD is within the zero-motion exit's threshold: the residual is quantisation noise, there is nothing to code.
//  * SIDE_CAP (B2V_FLAG_SIZE_CAP): its prediction and vector word into f.cap_pred and f.cap_mv, from which k_requant codes it again at a coarser QP.
// Whichever path chose the prediction, t.pred_y holds it here.
constexpr int SIDE_COST = 1, SIDE_CAP = 2;      // SIDE: f.scut is set, f.cap is set
template <bool WIDE, int SIDE>
__device__ __forceinline__ void finish_mb(const FrameCtx& f, MbTile& t, int lane, const MbPos& p, int qp, int ylo, int yhi, int mvx, int mvy, uint32_t uv_coloc, bool ltr = false) {
  const bool ref1 = ltr && mvx == LTR_MV;
  const size_t ysz = (size_t)f.cw * f.ch;
  if (SIDE & SIDE_COST) {      // first, while little is live (t.pred_y was written by other lanes: __syncwarp)
    __syncwarp();
    const int r8 = lane >> 1, c8 = (lane & 1) * 8;
    const uint2 c = *reinterpret_cast<const uint2*>(&t.cur_y[r8][c8]), pr = *reinterpret_cast<const uint2*>(&t.pred_y[r8][c8]);
    const int sad = __reduce_add_sync(FULL, (int)sad4acc(c.x, pr.x, sad4acc(c.y, pr.y, 0u)));
    const int vx = ref1 ? 0 : mvx, vy = ref1 ? 0 : mvy;
    const int lambda = me_lambda[qp];
    if (lane == 0) f.scut_cost[p.mb] = sad <= ME_EARLY_SAD_PER_LAMBDA * lambda ? 0 : sad + lambda * (se_bits_dev(vx) + se_bits_dev(vy) + (((vx | vy) & 3) ? ME_FRAC_PENALTY_BITS : 0));
  }

  const uint8_t* __restrict__ ref_uv = f.ref + ysz;
  const int rc4 = lane >> 2, cc4 = (lane & 3) * 4;
  const int mb = p.mb, mbx = p.mbx, mby = p.mby;
  {
    // chroma: mvC = luma mv, in 1/8 chroma samples (8.4.1.4, 8.4.2.2.2)
    const int xi = ref1 ? 0 : mvx >> 3, yi = ref1 ? 0 : mvy >> 3, xf = mvx & 7, yf = mvy & 7;
    const int cwc = f.cw >> 1;
    const int ya = clip3i(ylo >> 1, yhi >> 1, mby * 8 + yi + rc4), yb = clip3i(ylo >> 1, yhi >> 1, mby * 8 + yi + rc4 + 1);
    uint32_t out = 0;
    if (ref1) out = __ldg(reinterpret_cast<const uint32_t*>(f.lt + ysz + (size_t)(mby * 8 + rc4) * f.cw + mbx * 16 + cc4));   // long-term, zero vector
    else if ((mvx | mvy) == 0) out = uv_coloc;      // zero vector: the co-located pairs, loaded with the first batch
    else if ((xf | yf) == 0) {     // full-sample chroma position (most scrolling content): the (Cb,Cr) pairs are copied
#pragma unroll
      for (int px = 0; px < 2; px++) {
        const int xa = clip3i(0, cwc - 1, mbx * 8 + xi + (lane & 3) * 2 + px);
        out |= (uint32_t)__ldg(reinterpret_cast<const uint16_t*>(ref_uv + (size_t)ya * f.cw + xa * 2)) << (16 * px);
      }
    } else
#pragma unroll
    for (int px = 0; px < 2; px++) {
      const int x = (lane & 3) * 2 + px;
      const int xa = clip3i(0, cwc - 1, mbx * 8 + xi + x), xb = clip3i(0, cwc - 1, mbx * 8 + xi + x + 1);
#pragma unroll
      for (int k = 0; k < 2; k++) {
        const int A = __ldg(ref_uv + (size_t)ya * f.cw + xa * 2 + k), B = __ldg(ref_uv + (size_t)ya * f.cw + xb * 2 + k);
        const int C = __ldg(ref_uv + (size_t)yb * f.cw + xa * 2 + k), D = __ldg(ref_uv + (size_t)yb * f.cw + xb * 2 + k);
        const int v = ((8 - xf) * (8 - yf) * A + xf * (8 - yf) * B + (8 - xf) * yf * C + xf * yf * D + 32) >> 6;
        out |= (uint32_t)v << (8 * (px * 2 + k));
      }
    }
    *reinterpret_cast<uint32_t*>(&t.pred_uv[rc4][cc4]) = out;
  }
  __syncwarp();

  // ---- residual + reconstruction ------------------------------------------------------------------------
  // the vector as MbInfo's first word and the macroblock index are all that stays live across the transform: anything more
  // spills inside it at k_inter_lean's 64 registers.  So ref_idx 1 travels as a vector no macroblock can have, LTR_MV_WORD.
  const uint32_t mv = ref1 ? LTR_MV_WORD : (uint32_t)(mvx & 0xffff) | ((uint32_t)mvy << 16);
  if (SIDE & SIDE_CAP) {
    uint8_t* d = f.cap_pred + (size_t)mb * 384;
    *reinterpret_cast<uint2*>(d + (lane >> 1) * 16 + (lane & 1) * 8) = *reinterpret_cast<const uint2*>(&t.pred_y[lane >> 1][(lane & 1) * 8]);
    reinterpret_cast<uint32_t*>(d + 256)[lane] = reinterpret_cast<const uint32_t*>(&t.pred_uv[0][0])[lane];
    if (lane == 0) f.cap_mv[mb] = mv;
  }
  code_p_mb<WIDE>(f, t, lane, mb, qp, mv, ltr, ysz);
}

// The residual of P macroblock mb, whose source and prediction are in the tile, at `qp`; the I_PCM fallback; its reconstruction and
// record.  mv: finish_mb's vector word.  finish_mb, and k_requant at a picture's QP'.
template <bool WIDE>
__device__ __forceinline__ void code_p_mb(const FrameCtx& f, MbTile& t, int lane, int mb, int qp, uint32_t mv, bool ltr, size_t ysz) {
  int luma_bits, chroma_bits;
  int cbp = transform_mb<false>(t, lane, qp, f.coef + (size_t)mb * COEF_BLOCKS * 16, f.nnz + (size_t)mb * 32, luma_bits, chroma_bits);
  if ((WIDE ? 48 + WM_MVD_BITS : 48) + luma_bits + chroma_bits > MB_BITS_LIMIT) { apply_pcm(t, lane, f.nnz + (size_t)mb * 32); cbp = -1; }   // A.3.1: send raw
  __syncwarp();
  {
    const int ry = mb / f.mbw;
    store_recon(f, t, lane, (mb - ry * f.mbw) * 16, ry, ysz);
    if (lane == 0) {
      MbInfo mi; mi.mvx = (int16_t)(mv & 0xffff); mi.mvy = (int16_t)(mv >> 16); mi.type = MB_P16; mi.i16_mode = 0; mi.chroma_mode = 0; mi.cbp = (uint8_t)cbp;
      if (ltr && mv == LTR_MV_WORD) { mi.mvx = 0; mi.mvy = 0; mi.i16_mode = 1; }
      if (cbp < 0) { mi.mvx = 0; mi.mvy = 0; mi.type = MB_PCM; mi.cbp = 0; }   // too big for CAVLC: I_PCM (transform_mb)
      f.mbinfo[mb] = mi;
    }
  }
}

// Pass A: one warp per macroblock, raster order.  The macroblocks that leave motion estimation through the zero vector or through
// a temporal-predictor hit that needs no refinement are finished here; every other one goes into a queue for k_inter_search —
// anchors into the anchor queue, the rest into the other.  No search and no 48 x 48 window: the registers and shared memory of
// the search do not cap the occupancy of the common case.
// LTR (B2V_FLAG_LONG_TERM_REF): the block counts changed(k) for k_ltr_mark, and while a long-term picture is a reference, a
// macroblock that both exits fail is tested at the zero vector in it before it is queued (DESIGN.md §5.13).
// SIDE: every macroblock it finishes stores what B2V_FLAG_SCENE_CUT and B2V_FLAG_SIZE_CAP need of it (finish_mb).
template <bool SCALE, bool WIDE, bool LTR, int SIDE>
__device__ __forceinline__ void inter_lean(const FrameCtx& f) {
  __shared__ __align__(16) LeanSm sm_all[WARPS_PER_BLOCK];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int mbs = f.mbw * f.mbh;
  const int m = blockIdx.x * WARPS_PER_BLOCK + warp;
  if (!LTR && m >= mbs) return;
  const MbPos p = mb_pos(f, m);
  LeanSm& sm = sm_all[warp];
  MbTile& t = sm.t;
  const int qp = frame_qp(f), lambda = me_lambda[qp];
  const int ylo = p.band_r0 * 16, yhi = min(f.mbh, p.band_r0 + f.band_rows) * 16 - 1;
  MbStart s;
  if (LTR) {     // every warp of the block reaches the count, those past the last macroblock included
    if (m < mbs) s = start_mb<SCALE>(f, t, lane, p);
    const int n = __syncthreads_count(m < mbs && lane == 0 && s.sad0 > ME_EARLY_SAD_PER_LAMBDA * lambda);
    if (threadIdx.x == 0 && n) atomicAdd(&f.ltr->changed[f.pic & 1], n);
    if (m >= mbs) return;
  } else s = start_mb<SCALE>(f, t, lane, p);
  __syncwarp();
  // B2V_FLAG_LONG_TERM_REF: the zero vector into the long-term picture, while there is one.  Its SAD is taken here, where little
  // else is live, and used only if both exits below fail.
  bool lt_hit = false;
  if (LTR && s.sad0 > ME_EARLY_SAD_PER_LAMBDA * lambda && f.ltr->epoch == f.ltr_epoch) {
    const int r8 = lane >> 1, c8 = (lane & 1) * 8;
    const uint2 lz = __ldg(reinterpret_cast<const uint2*>(f.lt + (size_t)(p.mby * 16 + r8) * f.cw + p.mbx * 16 + c8));
    const uint2 c = *reinterpret_cast<const uint2*>(&t.cur_y[r8][c8]);
    lt_hit = __reduce_add_sync(FULL, (int)sad4acc(c.x, lz.x, sad4acc(c.y, lz.y, 0u))) <= ME_EARLY_SAD_PER_LAMBDA * lambda;
  }

  // zero-motion early termination: co-located block within the quantisation noise of this QP
  int mvx = 0, mvy = 0, sad_int = 0;
  if (s.sad0 <= ME_EARLY_SAD_PER_LAMBDA * lambda) {
    *reinterpret_cast<uint2*>(&t.pred_y[lane >> 1][(lane & 1) * 8]) = s.z;
  } else {
    // the temporal predictor on the part of the window around it.  A picture-edge macroblock, which needs per-sample clamping, is
    // deferred.
    const TemporalPred tp = temporal_predictor<WIDE>(s.prev);
    bool hit = false;
    if (tp.try_pred && (WIDE ? window_inside(f, p, tp.wx) : p.inside)) {
      const WinView w{&sm.pw[0][0], PW_WORDS, tp.ra, tp.wa};
      stage_pred_window(f, w, lane, p, ylo, yhi, tp);
      uint32_t best;
      // a hit whose previous vector was fractional is refined: k_inter_search does that
      hit = test_candidate(w, t, lane, tp.cdx, tp.cdy, lambda, s.sad0, best, tp.wx, tp.wy) && ((s.prev.mvx | s.prev.mvy) & 3) == 0;
      if (hit) {
        full_sample_pred(w, t, lane, 16 + tp.cdx, 16 + tp.cdy);
        mvx = 4 * (tp.wx + tp.cdx); mvy = 4 * (tp.wy + tp.cdy);
        sad_int = key_sad(best, lambda, mvx, mvy);
      }
    }
    // the long-term picture at the zero vector, under the zero-motion threshold (tested above): the macroblock is finished from it
    // (refIdx 1) and leaves the zero vector to its group and to the next picture, as a zero-vector exit does.  k_inter_search never
    // tries it.
    if (LTR && !hit && lt_hit) {
      const int r8 = lane >> 1, c8 = (lane & 1) * 8;
      *reinterpret_cast<uint2*>(&t.pred_y[r8][c8]) = __ldg(reinterpret_cast<const uint2*>(f.lt + (size_t)(p.mby * 16 + r8) * f.cw + p.mbx * 16 + c8));
      mvx = mvy = LTR_MV; hit = true;
    }
    if (!hit) {
      if (lane == 0) {
        const int qi = p.anchor ? 0 : 1;
        f.me_queue[2 + qi * mbs + atomicAdd(&f.me_queue[qi], 1)] = m;
      }
      return;
    }
  }
  if (p.anchor && lane == 0) publish_anchor<WIDE>(f, m, sad_int, LTR && mvx == LTR_MV ? 0 : mvx, LTR && mvy == LTR_MV ? 0 : mvy);   // sad_int 0 for refIdx 1
  finish_mb<WIDE, SIDE>(f, t, lane, p, qp, ylo, yhi, mvx, mvy, s.uv_coloc, LTR);
}
// CUT: B2V_FLAG_SCENE_CUT; the _cap variant: B2V_FLAG_SIZE_CAP
template <bool SCALE, bool WIDE, bool LTR, bool CUT>
__global__ void __launch_bounds__(32 * WARPS_PER_BLOCK, 8) k_inter_lean(FrameCtx f) { inter_lean<SCALE, WIDE, LTR, CUT ? SIDE_COST : 0>(f); }
template <bool SCALE, bool WIDE, bool LTR, bool CUT>
__global__ void __launch_bounds__(32 * WARPS_PER_BLOCK, 8) k_inter_lean_cap(FrameCtx f) { inter_lean<SCALE, WIDE, LTR, SIDE_CAP | (CUT ? SIDE_COST : 0)>(f); }

// One macroblock that k_inter_lean queued, from the start, through the same functions on the same inputs (source, reference and the
// previous picture's records are not written during the analysis of a picture).  Its co-located block failed the zero-motion test
// there and fails it again here, so that test is not repeated; its temporal predictor fails, or hits, as it did there.
// WIDE (B2V_FLAG_WIDE_MOTION): sm.win may hold the window centred on a full-sample vector (wx, wy) other than (0, 0) — a temporal or
// anchor predictor outside the co-located window's test range, or an anchor's coarse vector x 4; candidate indices and (dx, dy) are
// relative to that centre, costs are those of the real vector.
template <bool SCALE, bool WIDE, int SIDE>
__device__ __forceinline__ void search_mb(const FrameCtx& f, InterSm& sm, int lane, const MbPos& p) {
  const int mb = p.mb, x0 = p.mbx * 16, y0 = p.mby * 16;
  const bool anchor = p.anchor;
  MbTile& t = sm.t;
  const WinView win{&sm.win[0][0], WIN_WORDS, 0, 0};
  const int qp = frame_qp(f), lambda = me_lambda[qp];
  // reference rows this macroblock may touch: its own band (the band's decoder pads at the band's edges, 8.4.2.2.1)
  const int ylo = p.band_r0 * 16, yhi = min(f.mbh, p.band_r0 + f.band_rows) * 16 - 1;
  const uint8_t* __restrict__ ref_y = f.ref;
  const MbStart s = start_mb<SCALE>(f, t, lane, p);
  *reinterpret_cast<uint2*>(&sm.win[16 + (lane >> 1)][4 + (lane & 1) * 2]) = s.z;     // the co-located block: window rows 16..31, words 4..7
  __syncwarp();

  // ---- the reference.  A macroblock that carries a vector from the previous picture first gets only what the temporal-predictor
  // test, the refinement around it and the final prediction can touch — 24 rows x 8 words around the predicted position instead of
  // the 48 x 12 window; the rest follows only if the predictor is rejected and the search has to run.
  const TemporalPred tp = temporal_predictor<WIDE>(s.prev);
  bool window_complete = false;     // sm.win holds the whole co-located window
  int wx = 0, wy = 0;               // WIDE: the centre of the window sm.win holds
  // WIDE: the whole window centred on (cx, cy), centre block included; (0, 0) restores the co-located window after another
  auto stage_at = [&](int cx, int cy) {
    if (window_inside(f, p, cx)) {
      const uint32_t* base = reinterpret_cast<const uint32_t*>(ref_y + x0 - 16 + cx);
      for (int i = lane; i < WIN_ROWS * WIN_WORDS; i += 32) {
        const int row = i / WIN_WORDS, w = i - row * WIN_WORDS;
        sm.win[row][w] = __ldg(base + (size_t)clip3i(ylo, yhi, y0 - 16 + cy + row) * (f.cw >> 2) + w);
      }
    } else {
      for (int i = lane; i < WIN_ROWS * WIN_WORDS; i += 32) {
        const int row = i / WIN_WORDS, w = i - row * WIN_WORDS;
        const uint8_t* rr = ref_y + (size_t)clip3i(ylo, yhi, y0 - 16 + cy + row) * f.cw;
        uint32_t v = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) v |= (uint32_t)__ldg(rr + clip3i(0, f.cw - 1, x0 - 16 + cx + w * 4 + k)) << (8 * k);
        sm.win[row][w] = v;
      }
    }
    wx = cx; wy = cy;
    window_complete = (cx | cy) == 0;
    __syncwarp();
  };
  auto stage_window = [&]() {
    if (WIDE && (wx | wy)) stage_at(0, 0);
    else if (p.inside) {   // 512 more words: lanes 0..23 take (row pair j, word) = two rows of 12 words per step — no index arithmetic
      // beyond an add per step —, every load issued before the first shared-memory store
      uint32_t v[24];
      const int half = lane >= 12 ? 1 : 0, w = lane - 12 * half;
      const bool mid = w >= 4 && w < 8;
      const uint32_t* base = reinterpret_cast<const uint32_t*>(ref_y + x0 - 16) + w;
      if (lane < 24) {
#pragma unroll
        for (int j = 0; j < 24; j++) {
          const int row = 2 * j + half;
          const bool centre = j >= 8 && j < 16 && mid;
          v[j] = centre ? 0u : __ldg(base + (size_t)clip3i(ylo, yhi, y0 - 16 + row) * (f.cw >> 2));
        }
#pragma unroll
        for (int j = 0; j < 24; j++) {
          const bool centre = j >= 8 && j < 16 && mid;
          if (!centre) sm.win[2 * j + half][w] = v[j];
        }
      }
    } else {   // picture edge: per-sample clamping (8.4.2.2.1 reference sample padding)
      for (int i = lane; i < WIN_ROWS * WIN_WORDS; i += 32) {
        const int row = i / WIN_WORDS, w = i - row * WIN_WORDS;
        if (row >= 16 && row < 32 && w >= 4 && w < 8) continue;
        const uint8_t* rr = ref_y + (size_t)clip3i(ylo, yhi, y0 - 16 + row) * f.cw;
        uint32_t v = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) v |= (uint32_t)__ldg(rr + clip3i(0, f.cw - 1, x0 - 16 + w * 4 + k)) << (8 * k);
        sm.win[row][w] = v;
      }
    }
    window_complete = true;
    __syncwarp();
  };
  // k_inter_lean did not test the predictor of a picture-edge macroblock: it is tested here, on the full clamped window
  if (WIDE && tp.try_pred && (tp.wx | tp.wy)) stage_at(tp.wx, tp.wy);
  else if (p.inside && tp.try_pred) stage_pred_window(f, win, lane, p, ylo, yhi, tp); else stage_window();
  // ---- temporal predictor; quarter-sample refinement then runs as after a search ----
  uint32_t best = 0xffffffffu;
  bool pred_frac = false, reduced = false;
  if (tp.try_pred && test_candidate(win, t, lane, tp.cdx, tp.cdy, lambda, s.sad0, best, tp.wx, tp.wy)) pred_frac = ((s.prev.mvx | s.prev.mvy) & 3) != 0;
  // ---- anchor predictor (oracle/h264_ref.c encode_inter_mb): the temporal predictor failed (or there was none) — motion that
  // STARTS in this picture.  Instead of one exhaustive search per macroblock, try what this group's anchor has found. ----
  if (best == 0xffffffffu && !anchor) {
    // written by k_inter_lean or by the anchor pass, both earlier in stream order.  The tag is always there; were it missing, the
    // macroblock would run the exhaustive search and the stream would differ from the oracle's.
    const unsigned long long v = f.me_pub[(size_t)p.ay * f.mbw + p.ax];
    const bool have = (uint32_t)(v >> 32) == (uint32_t)f.pic + 1u;
    const int amvx = WIDE ? (int)(uint32_t)v >> 20 : (int)(int8_t)(v >> 8), amvy = WIDE ? (int)((uint32_t)v << 20) >> 20 : (int)(int8_t)v;
    int kx, ky;
    bool in_window = full_sample_candidate(amvx, amvy, kx, ky);
    int ox = 0, oy = 0;
    if (WIDE && have && !in_window && mv_ok(kx, ky)) {     // far: the window centred on it, as for a far temporal predictor
      ox = kx & ~3; oy = ky; kx -= ox; ky -= oy; in_window = true;
      stage_at(ox, oy);
    } else if (!window_complete) stage_window();   // any candidate position may be tried; needed by the search anyway if it is rejected
    // (ox, oy) = (0, 0) for the zero vector: in a shifted window the test below cannot be the zero vector's
    const bool zero_again = ((ox + kx) | (oy + ky)) == 0 && tp.try_pred && ((tp.wx + tp.cdx) | (tp.wy + tp.cdy)) == 0;      // the zero vector is not tested twice
    if (have && !zero_again && in_window && test_candidate(win, t, lane, kx, ky, lambda, s.sad0, best, ox, oy)) pred_frac = ((amvx | amvy) & 3) != 0;
    // new content: the anchor's exhaustive search found nothing (bit 16) and the co-located block is as far off — the search
    // shrinks to the rows around dy = 0: picking the least bad of 1089 noise candidates buys hardly more than picking it of 160
    else reduced = have && ((v >> 16) & 1) != 0 && s.sad0 >= ME_REFINE_MAX_SAD;
  }
  const bool searched = best == 0xffffffffu;
  if (searched && !window_complete) stage_window();          // predictor rejected: the search needs the whole window
  if (searched) best = reduced ? search_rows<ME_NEWCONTENT_DY>(sm, lane, lambda) : search_rows<16>(sm, lane, lambda);
  // WIDE, an anchor that searched: the same search in the window centred on its group's coarse vector x 4 (k_coarse), unless the
  // co-located search covered that vector with the 4 samples either way one decimated sample spans.  The cheaper result by true cost
  // wins, the co-located window on equal cost (keys of two windows are compared by cost alone: their indices are window-relative).
  if (WIDE && searched && anchor) {
    const int cv = f.coarse[mb];
    const int cx = 4 * (int)(int16_t)(cv & 0xffff), cy = 4 * (cv >> 16);
    if (cv != COARSE_NONE && (cx < -12 || cx > 11 || cy < -12 || cy > 12)) {
      const uint32_t best0 = best;
      stage_at(cx, cy);
      const uint32_t best1 = search_rows<16, true>(sm, lane, lambda, cx, cy);
      if ((best1 >> 11) < (best0 >> 11)) best = best1; else stage_window();
    }
  }
  const int dyi = (best & 2047) >> 5, dxi = best & 31, dx = dxi - 16, dy = dyi - 16;

  // ---- quarter-sample refinement (DESIGN.md §5.3; oracle/h264_ref.c encode_inter_mb) ---------------------------------
  int mvx = 4 * (wx + dx), mvy = 4 * (wy + dy);
  // refine only inside the window (6-tap support [-3,+18]) and when the full-sample match is not already within the
  // quantisation noise of this QP (same threshold as the zero-motion early termination)
  const int sad_int = key_sad(best, lambda, mvx, mvy);
  // a predictor hit whose previous vector was full-sample is not refined again: the previous refinement already preferred it
  // ... and not when the full-sample match is hopeless (mean absolute difference >= 32 per sample: new content, nothing to polish —
  // the refinement is a third of the work of a searched macroblock and bought 0 % bits on such pictures)
  const bool refine = (searched || pred_frac) && abs(dx) <= 13 && abs(dy) <= 13 && sad_int > ME_EARLY_SAD_PER_LAMBDA * lambda && sad_int < ME_REFINE_MAX_SAD;
  const int ox = dxi, oy = dyi;                                        // window coordinates of the full-sample position
  if (refine) {
    // half-sample planes
    for (int i = lane; i < 22 * 17; i += 32) {
      const int v = i / 17, u = i - v * 17;                             // row Y = v-3, column X = u-1
      const uint8_t* g = reinterpret_cast<const uint8_t*>(&sm.win[oy + v - 3][0]) + ox + u - 1;
      sm.b1[v][u] = (int16_t)((int)g[-2] - 5 * (int)g[-1] + 20 * (int)g[0] + 20 * (int)g[1] - 5 * (int)g[2] + (int)g[3]);
    }
    for (int i = lane; i < 17 * 18; i += 32) {
      const int v = i / 18, u = i - v * 18;                             // Y = v-1, X = u-1
      const uint8_t* g = reinterpret_cast<const uint8_t*>(&sm.win[oy + v - 1][0]) + ox + u - 1;
      const int h1 = (int)g[-2 * 48] - 5 * (int)g[-48] + 20 * (int)g[0] + 20 * (int)g[48] - 5 * (int)g[2 * 48] + (int)g[3 * 48];
      sm.hq[v][u] = (uint8_t)clip255((h1 + 16) >> 5);
    }
    __syncwarp();
    for (int i = lane; i < 18 * 17; i += 32) {
      const int v = i / 17, u = i - v * 17;                             // Y = v-1 -> b1 row v+2
      sm.bq[v][u] = (uint8_t)clip255(((int)sm.b1[v + 2][u] + 16) >> 5);
    }
    for (int i = lane; i < 17 * 17; i += 32) {
      const int v = i / 17, u = i - v * 17;                             // Y = v-1 -> b1 rows v..v+5
      const int j1 = (int)sm.b1[v][u] - 5 * (int)sm.b1[v + 1][u] + 20 * (int)sm.b1[v + 2][u] + 20 * (int)sm.b1[v + 3][u] - 5 * (int)sm.b1[v + 4][u] + (int)sm.b1[v + 5][u];
      sm.jq[v][u] = (uint8_t)clip255((j1 + 512) >> 10);
    }
    __syncwarp();
    // stage H (half-sample neighbours), stage Q (quarter-sample neighbours of the stage-H winner)
    int cx = 0, cyq = 0;
    uint32_t centre_cost = best >> 11;
    const int half = lane >> 4, row = lane & 15;
    const uint4 cur4 = *reinterpret_cast<const uint4*>(&t.cur_y[row][0]);
#pragma unroll 1
    for (int stage = 0; stage < 2; stage++) {
      const int step = stage == 0 ? 2 : 1;
      uint32_t bestk = (centre_cost << 4);                              // candidate 0 = centre
#pragma unroll 1
      for (int k = 0; k < 4; k++) {
        const int cand = 2 * k + half;                                  // 0..7 in the order of nb8[]
        const int nx = cand < 3 ? cand - 1 : cand == 3 ? -1 : cand == 4 ? 1 : cand - 6;
        const int ny = cand < 3 ? -1 : cand < 5 ? 0 : 1;
        const int qx = cx + nx * step, qy = cyq + ny * step;
        uint32_t pr[4];
        subpel_row(sm, ox, oy, qx, qy, row, pr);
        int sad = (int)sad4acc(cur4.x, pr[0], sad4acc(cur4.y, pr[1], sad4acc(cur4.z, pr[2], sad4acc(cur4.w, pr[3], 0u))));
        sad += __shfl_xor_sync(FULL, sad, 1); sad += __shfl_xor_sync(FULL, sad, 2);
        sad += __shfl_xor_sync(FULL, sad, 4); sad += __shfl_xor_sync(FULL, sad, 8);
        const uint32_t cost = (uint32_t)(sad + lambda * (se_bits_dev(4 * (wx + dx) + qx) + se_bits_dev(4 * (wy + dy) + qy) + (((qx | qy) & 3) ? ME_FRAC_PENALTY_BITS : 0)));
        uint32_t key = (cost << 4) | (uint32_t)(cand + 1);
        key = min(key, __shfl_xor_sync(FULL, key, 16));
        bestk = min(bestk, key);
      }
      const int bi = bestk & 15;
      if (bi) {
        const int cand = bi - 1;
        cx += (cand < 3 ? cand - 1 : cand == 3 ? -1 : cand == 4 ? 1 : cand - 6) * step;
        cyq += (cand < 3 ? -1 : cand < 5 ? 0 : 1) * step;
        centre_cost = bestk >> 4;
      }
    }
    mvx += cx; mvy += cyq;
    if (lane < 16) {
      uint32_t pr[4];
      subpel_row(sm, ox, oy, cx, cyq, lane, pr);
      *reinterpret_cast<uint4*>(&t.pred_y[lane][0]) = make_uint4(pr[0], pr[1], pr[2], pr[3]);
    }
  }
  if (anchor && lane == 0) publish_anchor<WIDE>(f, mb, sad_int, mvx, mvy);
  if (!refine) full_sample_pred(win, t, lane, dxi, dyi);
  finish_mb<WIDE, SIDE>(f, t, lane, p, qp, ylo, yhi, mvx, mvy, s.uv_coloc);
}

// Passes B and C: the queue k_inter_lean filled (0: anchors, 1: the rest), walked by a grid of the kernel's resident capacity.  No
// decision here depends on another entry of the same queue, so the order inside a queue does not matter.
template <bool SCALE, bool WIDE, int SIDE>
__device__ __forceinline__ void inter_search(const FrameCtx& f, int queue) {
  __shared__ __align__(16) InterSm sm_all[WARPS_PER_BLOCK];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = f.me_queue[queue];
  const int* q = f.me_queue + 2 + (size_t)queue * f.mbw * f.mbh;
  for (int i = blockIdx.x * WARPS_PER_BLOCK + warp; i < n; i += gridDim.x * WARPS_PER_BLOCK) {
    search_mb<SCALE, WIDE, SIDE>(f, sm_all[warp], lane, mb_pos(f, q[i]));
    __syncwarp();
  }
}
template <bool SCALE, bool WIDE, bool CUT>
__global__ void __launch_bounds__(32 * WARPS_PER_BLOCK, 5) k_inter_search(FrameCtx f, int queue) { inter_search<SCALE, WIDE, CUT ? SIDE_COST : 0>(f, queue); }
template <bool SCALE, bool WIDE, bool CUT>
__global__ void __launch_bounds__(32 * WARPS_PER_BLOCK, 5) k_inter_search_cap(FrameCtx f, int queue) {
  inter_search<SCALE, WIDE, SIDE_CAP | (CUT ? SIDE_COST : 0)>(f, queue);
}

// ---- k_requant (B2V_FLAG_SIZE_CAP): P picture k once more at the QP' k_size_cap chose, when it chose one; one warp per macroblock ----
// Every macroblock keeps the prediction and vector the analysis stored (finish_mb) and is coded again from them by the code the
// analysis ran (code_p_mb): transform, quantisation, the I_PCM fallback in both directions, reconstruction, levels, nnz, record.
// The second CAVLC pass then evaluates P_Skip again.  oracle/h264_cap_ref.c requant.
constexpr int REQUANT_WARPS = 4;
__global__ void __launch_bounds__(32 * REQUANT_WARPS) k_requant(FrameCtx f) {
  if (!*reinterpret_cast<const volatile int32_t*>(&f.cap->recode[f.pic & 1])) return;
  __shared__ __align__(16) MbTile tiles[REQUANT_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int mb = blockIdx.x * REQUANT_WARPS + warp;
  if (mb >= f.mbw * f.mbh) return;
  MbTile& t = tiles[warp];
  const size_t ysz = (size_t)f.cw * f.ch;
  const int mby = mb / f.mbw, mbx = mb - mby * f.mbw;
  stage_source(f, t, lane, mbx * 16, mby, ysz);
  const uint8_t* d = f.cap_pred + (size_t)mb * 384;
  *reinterpret_cast<uint2*>(&t.pred_y[lane >> 1][(lane & 1) * 8]) = *reinterpret_cast<const uint2*>(d + (lane >> 1) * 16 + (lane & 1) * 8);
  reinterpret_cast<uint32_t*>(&t.pred_uv[0][0])[lane] = reinterpret_cast<const uint32_t*>(d + 256)[lane];
  const uint32_t mv = f.cap_mv[mb];
  const int qp = f.cap->qp[f.pic & 1];
  __syncwarp();
  if (f.wide) code_p_mb<true>(f, t, lane, mb, qp, mv, f.ltr != nullptr, ysz);
  else code_p_mb<false>(f, t, lane, mb, qp, mv, f.ltr != nullptr, ysz);
}

int launch_requant(const FrameCtx& f, cudaStream_t st) {
  k_requant<<<(f.mbw * f.mbh + REQUANT_WARPS - 1) / REQUANT_WARPS, 32 * REQUANT_WARPS, 0, st>>>(f);
  return 1;
}

cudaError_t inter_search_grid(int* blocks) {
  int dev = 0, sms = 0, per_sm = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_inter_search<false, false, false>, 32 * WARPS_PER_BLOCK, 0);
  *blocks = sms * per_sm;
  return e;
}

// The three passes of a P picture: SCALE, the previous picture's vectors span another reference distance than this picture's
// (B2V_FLAG_DROPPABLE); WIDE, B2V_FLAG_WIDE_MOTION (k_coarse ran first on this stream); LTR, B2V_FLAG_LONG_TERM_REF; CUT,
// B2V_FLAG_SCENE_CUT (k_scene_cut follows); CAP, B2V_FLAG_SIZE_CAP (k_size_cap follows).
template <bool SCALE, bool WIDE, bool LTR, bool CUT, bool CAP>
void launch_passes(const FrameCtx& f, int lean_blocks, cudaStream_t st) {
  if (CAP) {
    k_inter_lean_cap<SCALE, WIDE, LTR, CUT><<<lean_blocks, 32 * WARPS_PER_BLOCK, 0, st>>>(f);
    k_inter_search_cap<SCALE, WIDE, CUT><<<f.search_blocks, 32 * WARPS_PER_BLOCK, 0, st>>>(f, 0);
    k_inter_search_cap<SCALE, WIDE, CUT><<<f.search_blocks, 32 * WARPS_PER_BLOCK, 0, st>>>(f, 1);
    return;
  }
  k_inter_lean<SCALE, WIDE, LTR, CUT><<<lean_blocks, 32 * WARPS_PER_BLOCK, 0, st>>>(f);
  k_inter_search<SCALE, WIDE, CUT><<<f.search_blocks, 32 * WARPS_PER_BLOCK, 0, st>>>(f, 0);   // anchors
  k_inter_search<SCALE, WIDE, CUT><<<f.search_blocks, 32 * WARPS_PER_BLOCK, 0, st>>>(f, 1);   // the rest: read the anchors' vectors
}
template <bool CUT, bool CAP>
void launch_passes_for(const FrameCtx& f, int lean_blocks, cudaStream_t st) {
  // The long-term reference never comes with droppable pictures (check_coding_flags), so with it both distances are 1: LTR
  // implies !SCALE, and no <true, *, true, *> variant is compiled.
  const bool scale = f.ref_dist != f.prev_ref_dist;
  if (f.ltr) f.wide ? launch_passes<false, true, true, CUT, CAP>(f, lean_blocks, st) : launch_passes<false, false, true, CUT, CAP>(f, lean_blocks, st);
  else if (scale) f.wide ? launch_passes<true, true, false, CUT, CAP>(f, lean_blocks, st) : launch_passes<true, false, false, CUT, CAP>(f, lean_blocks, st);
  else f.wide ? launch_passes<false, true, false, CUT, CAP>(f, lean_blocks, st) : launch_passes<false, false, false, CUT, CAP>(f, lean_blocks, st);
}

int launch_inter(const FrameCtx& f, cudaStream_t st) {
  // both queues empty; the counters are only read by the two k_inter_search launches that follow
  cudaMemsetAsync(f.me_queue, 0, 2 * sizeof(int), st);
  const int lean_blocks = (f.mbw * f.mbh + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK;
  if (f.cap) f.scut ? launch_passes_for<true, true>(f, lean_blocks, st) : launch_passes_for<false, true>(f, lean_blocks, st);
  else f.scut ? launch_passes_for<true, false>(f, lean_blocks, st) : launch_passes_for<false, false>(f, lean_blocks, st);
  return 3;
}

// ---- k_coarse (B2V_FLAG_WIDE_MOTION): one block per anchor group (4 x 4 macroblocks, counted inside each band), every picture ----
//  1. the group's samples of this picture's decimated luma (each the rounded mean of a 4x4 block of the coded luma) into f.dec_cur,
//     the plane kept with the reconstruction buffer this picture writes (an IDR picture stops here);
//  2. the anchor's co-located SAD; at or below the early-termination threshold the group gets no coarse vector;
//  3. the group's decimated block (up to 16 x 16) against the reference picture's plane at dx in [-32, 31], dy in [-64, 63], every
//     position inside the picture and the band: 256 threads, each a column dx of 16 consecutive dy twice, 16 SADs in registers fed
//     row by row with VABSDIFF4 as search_rows does; the minimum of (SAD, |dx| + |dy|, dy, dx) as one 37-bit key.
// oracle/h264_wide_ref.c decimate, coarse_search.
constexpr int CO_ROWS = 2 * WM_DY + 16, CO_WORDS = (2 * WM_DX + 16) / 4 + 1;   // reference tile: decimated rows from Y0 - WM_DY, words from X0 - WM_DX (zero outside)
__global__ void __launch_bounds__(256) k_coarse(FrameCtx f) {
  __shared__ __align__(16) uint32_t tile[CO_ROWS][CO_WORDS];
  __shared__ __align__(16) uint8_t cur[16][16];
  __shared__ unsigned long long s_best;
  __shared__ int s_sad0;
  const int tid = threadIdx.x;
  const int gpb = (f.band_rows + 3) >> 2;                      // group rows per band
  const int band = blockIdx.y / gpb;
  const int br0 = band * f.band_rows, br1 = min(f.mbh, br0 + f.band_rows), gy0 = br0 + 4 * (blockIdx.y - band * gpb);
  if (gy0 >= br1) return;
  const int gx0 = 4 * blockIdx.x, gx1 = min(gx0 + 4, f.mbw), gy1 = min(gy0 + 4, br1);
  const int dw = f.cw >> 2, X0 = 4 * gx0, Y0 = 4 * gy0, W = 4 * (gx1 - gx0), H = 4 * (gy1 - gy0);
  {
    const int r = tid >> 4, c = tid & 15;
    uint32_t d = 0;
    if (r < H && c < W) {
      const uint8_t* src = f.cur + (size_t)(4 * (Y0 + r)) * f.cw + 4 * (X0 + c);
      uint32_t sum = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) sum += __vsadu4(*reinterpret_cast<const uint32_t*>(src + (size_t)k * f.cw), 0u);
      d = (sum + 8) >> 4;
      f.dec_cur[(size_t)(Y0 + r) * dw + X0 + c] = (uint8_t)d;
    }
    cur[r][c] = (uint8_t)d;                                    // zero outside the group: those bytes are masked below
  }
  if (f.idr) return;
  const int ax = min(gx0 + 1, f.mbw - 1), ay = min(gy0 + 1, br1 - 1), amb = ay * f.mbw + ax;
  if (tid == 0) { s_sad0 = 0; s_best = ~0ull; }
  __syncthreads();
  {
    const size_t o = (size_t)(ay * 16 + (tid >> 4)) * f.cw + ax * 16 + (tid & 15);
    const int d = __reduce_add_sync(FULL, abs((int)f.cur[o] - (int)f.ref[o]));
    if ((tid & 31) == 0) atomicAdd(&s_sad0, d);
  }
  __syncthreads();
  if (s_sad0 <= ME_EARLY_SAD_PER_LAMBDA * me_lambda[frame_qp(f)]) { if (tid == 0) f.coarse[amb] = COARSE_NONE; return; }
  const int ylo = 4 * br0, yhi = 4 * br1;                      // decimated rows of the band: [ylo, yhi)
  for (int i = tid; i < CO_ROWS * CO_WORDS; i += 256) {
    const int row = i / CO_WORDS, w = i - row * CO_WORDS;
    const int y = Y0 - WM_DY + row, x = X0 - WM_DX + 4 * w;          // x and dw are multiples of 4: a word lies inside or outside whole
    tile[row][w] = y >= ylo && y < yhi && x >= 0 && x < dw ? *reinterpret_cast<const uint32_t*>(f.dec_ref + (size_t)y * dw + x) : 0u;
  }
  __syncthreads();
  const int dxi = tid & 63, dx = dxi - WM_DX, nw = W >> 2, wi = dxi >> 2, sh = (dxi & 3) * 8;
  uint32_t c[16][4];
#pragma unroll
  for (int r = 0; r < 16; r++) {
    const uint4 v = *reinterpret_cast<const uint4*>(&cur[r][0]);
    c[r][0] = v.x; c[r][1] = v.y; c[r][2] = v.z; c[r][3] = v.w;
  }
  const bool x_ok = X0 + dx >= 0 && X0 + dx + W <= dw;
  unsigned long long best = ~0ull;
#pragma unroll 1
  for (int chunk = tid >> 6; chunk < 8; chunk += 4) {
    const int dy0 = -WM_DY + 16 * chunk;                       // this item: dy in [dy0, dy0 + 15], tile rows dy0 + WM_DY + k + r
    uint32_t acc[16];
#pragma unroll
    for (int k = 0; k < 16; k++) acc[k] = 0;
#pragma unroll
    for (int y = 0; y < 31; y++) {
      const uint32_t* wr = &tile[dy0 + WM_DY + y][wi];
      const uint32_t w0 = wr[0], w1 = wr[1], w2 = wr[2], w3 = wr[3], w4 = wr[4];
      const uint32_t a0 = __funnelshift_r(w0, w1, sh), a1 = nw > 1 ? __funnelshift_r(w1, w2, sh) : 0u;
      const uint32_t a2 = nw > 2 ? __funnelshift_r(w2, w3, sh) : 0u, a3 = nw > 3 ? __funnelshift_r(w3, w4, sh) : 0u;
#pragma unroll
      for (int r = 0; r < 16; r++) {
        const int k = y - r;
        if (k >= 0 && k < 16 && r < H) acc[k] = sad4acc(c[r][0], a0, sad4acc(c[r][1], a1, sad4acc(c[r][2], a2, sad4acc(c[r][3], a3, acc[k]))));
      }
    }
#pragma unroll
    for (int k = 0; k < 16; k++) {
      const int dy = dy0 + k;
      const unsigned long long key = (unsigned long long)acc[k] << 20 | (unsigned long long)(abs(dx) + abs(dy)) << 13 | (unsigned long long)(dy + 64) << 6 | (unsigned long long)dxi;
      if (x_ok && Y0 + dy >= ylo && Y0 + dy + H <= yhi) best = min(best, key);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(FULL, best, o));
  if ((tid & 31) == 0) atomicMin(&s_best, best);
  __syncthreads();
  if (tid == 0) {
    const unsigned long long b = s_best;
    f.coarse[amb] = b == ~0ull ? COARSE_NONE : (int)(((int)(b & 63) - 32) & 0xffff) | (int)((unsigned)((int)((b >> 6) & 127) - 64) << 16);
  }
}

int launch_coarse(const FrameCtx& f, cudaStream_t st) {
  const dim3 grid((f.mbw + 3) / 4, f.n_bands * ((f.band_rows + 3) / 4));
  k_coarse<<<grid, 256, 0, st>>>(f);
  return 1;
}

// ---- k_ltr_mark (B2V_FLAG_LONG_TERM_REF): once per P picture k, on the analysis stream behind the analysis (DESIGN.md §5.13) ----
// Picture k marks picture k-1 long-term when changed(k) >= max(ceil(mbs / 64), 8 * changed(k-1)): a large change right after a
// quiet picture (changed of an IDR picture = mbs).  Every block decides from the two counts, which nothing in this launch writes,
// and copies its share of f.ref (picture k-1's reconstruction) into f.lt when marking; block 0 records the decision for the entropy
// stage of picture k and, when marking, makes the long-term picture valid for picture k+1.  Picture k itself was analysed against
// the long-term picture as it stood: the marking takes effect after picture k (8.2.5).  oracle/h264_ltr_ref.c ltr_encode.
constexpr int LTR_CHANGED_MIN_DIV = 64, LTR_CHANGED_RATIO = 8;
constexpr int LTR_COPY_THREADS = 256;
__global__ void __launch_bounds__(LTR_COPY_THREADS) k_ltr_mark(FrameCtx f) {
  const int mbs = f.mbw * f.mbh;
  const int changed = f.ltr->changed[f.pic & 1], prev = f.prev_idr ? mbs : f.ltr->changed[(f.pic & 1) ^ 1];
  const bool mark = changed >= max((mbs + LTR_CHANGED_MIN_DIV - 1) / LTR_CHANGED_MIN_DIV, LTR_CHANGED_RATIO * prev);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const bool active = f.ltr->epoch == f.ltr_epoch;
    LtrPic r; r.active = active; r.mark = mark; r.drop_st = mark && !active; r.pad = 0;
    f.ltr->pic[f.pic & 1] = r;
    if (mark) f.ltr->epoch = f.ltr_epoch;
  }
  if (!mark) return;
  const size_t n16 = (size_t)f.cw * f.ch * 3 / 2 / 16;          // coded width is a multiple of 16
  const uint4* src = reinterpret_cast<const uint4*>(f.ref);
  uint4* dst = reinterpret_cast<uint4*>(f.lt);
  for (size_t i = (size_t)blockIdx.x * LTR_COPY_THREADS + threadIdx.x; i < n16; i += (size_t)gridDim.x * LTR_COPY_THREADS) dst[i] = __ldg(src + i);
}

int launch_ltr_mark(const FrameCtx& f, cudaStream_t st) {
  const size_t n16 = (size_t)f.cw * f.ch * 3 / 2 / 16;
  const size_t want = (n16 + 4 * LTR_COPY_THREADS - 1) / (4 * LTR_COPY_THREADS);   // four 16-byte words per thread, at most 8 blocks per SM
  const int blocks = (int)(want < 1056 ? want : 1056);
  k_ltr_mark<<<blocks, LTR_COPY_THREADS, 0, st>>>(f);
  return 1;
}

}  // namespace b2v
