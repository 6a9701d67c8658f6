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
// which reads the anchors' vectors.  Apart from that, there is no dependency between macroblocks of a P picture: motion-vector
// prediction and the P_Skip decision only matter for entropy coding and are resolved in h264_entropy.cu.
// Encoder decisions: DESIGN.md §5.3; CPU restatement: oracle/h264_ref.c encode_inter_mb().
#include "h264_common.cuh"
#include "h264_kernels.h"

namespace b2v {

constexpr int WIN_ROWS = 48, WIN_WORDS = 12;
constexpr int PW_ROWS = 24, PW_WORDS = 8;      // the part of the window around a temporal predictor (k_inter_lean)
constexpr int WARPS_PER_BLOCK = 4;
constexpr int ME_EARLY_SAD_PER_LAMBDA = 96;   // skip the search when SAD(0,0) <= 96 * lambda(qp)

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
  const uint32_t* p;
  int stride, r0, w0;
  __device__ __forceinline__ const uint32_t* at(int r, int w) const { return p + (r - r0) * stride + (w - w0); }
};

constexpr int ME_PRED_SAD_FACTOR = 4;      // temporal predictor accepted up to 4x the early-termination threshold (and only as a strict local minimum)
constexpr int ME_FRAC_PENALTY_BITS = 4;   // fractional vectors pay 4 extra bits in the refinement cost
constexpr int ME_REFINE_MAX_SAD = 8192;   // no sub-sample refinement of a full-sample match this bad
constexpr int ME_NEWCONTENT_DY = 2;       // vertical range of the reduced search on new content

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
template <int DYR>
__device__ __forceinline__ uint32_t search_rows(const InterSm& sm, int lane, int lambda) {
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
  const int bits_x = se_bits_c(4 * (lane - 16));
  uint32_t best = 0xffffffffu;
#pragma unroll
  for (int k = 0; k < N; k++) {
    const int dyi = k + Y0;                     // dy + 16
    const uint32_t cost = acc[k] + (uint32_t)(lambda * (bits_x + se_bits_c(4 * (dyi - 16))));
    best = min(best, (cost << 11) | (uint32_t)(dyi * 32 + lane));
  }
  return __reduce_min_sync(FULL, best);
}

// A macroblock's place: its band's first row and the anchor of its 4x4 group — one per group, at offset (1,1), groups counted inside
// each band (oracle/h264_ref.c anchor_of()).  An anchor's vector is the first candidate of the other macroblocks of its group whose
// temporal predictor failed.
struct MbPos {
  int mb, mbx, mby, band_r0, ax, ay;
  bool anchor;
};
__device__ __forceinline__ MbPos mb_pos(const FrameCtx& f, int mb) {
  MbPos p;
  p.mb = mb; p.mby = mb / f.mbw; p.mbx = mb - p.mby * f.mbw;
  p.band_r0 = p.mby / f.band_rows * f.band_rows;
  p.ax = min(4 * (p.mbx >> 2) + 1, f.mbw - 1);
  p.ay = p.band_r0 + min(4 * ((p.mby - p.band_r0) >> 2) + 1, min(f.mbh - p.band_r0, f.band_rows) - 1);
  p.anchor = p.ax == p.mbx && p.ay == p.mby;
  return p;
}

// the 16x16 source block and its chroma into the tile; returns this lane's 8 luma samples (row lane >> 1, columns (lane & 1) * 8 ..)
__device__ __forceinline__ uint2 stage_source(const FrameCtx& f, MbTile& t, int lane, int x0, int mby) {
  const int r8 = lane >> 1, c8 = (lane & 1) * 8;
  const uint2 v = *reinterpret_cast<const uint2*>(f.cur + (size_t)(mby * 16 + r8) * f.cw + x0 + c8);
  *reinterpret_cast<uint2*>(&t.cur_y[r8][c8]) = v;
  if (lane < 16) {
    const uint2 w = *reinterpret_cast<const uint2*>(f.cur + (size_t)f.cw * f.ch + (size_t)(mby * 8 + r8) * f.cw + x0 + c8);
    *reinterpret_cast<uint2*>(&t.cur_uv[r8][c8]) = w;
  }
  return v;
}

// ---- temporal-predictor early termination (DESIGN.md §5.3; oracle/h264_ref.c encode_inter_mb / try_candidate) ----
// Candidate (kx,ky), full samples, window staged around it: true (and `best` = its key) when its SAD is within 4x the noise
// threshold AND it is a strict local minimum of the cost over its 8 full-sample neighbours AND it costs no more than the zero vector.
__device__ __forceinline__ bool test_candidate(const WinView& w, const MbTile& t, int lane, int kx, int ky, int lambda, int sad0, uint32_t& best) {
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
      const uint32_t cost = (uint32_t)(sad + lambda * (se_bits_dev(4 * (kx + i)) + se_bits_dev(4 * (ky + j))));
      const uint32_t key = (cost << 11) | (uint32_t)((ky + j + 16) * 32 + (kx + i + 16));
      if (i == 0 && j == 0) kc = key; else kmin = min(kmin, key);
    }
  }
  const int sadc = (int)(kc >> 11) - lambda * (se_bits_dev(4 * kx) + se_bits_dev(4 * ky));
  const uint32_t key0 = ((uint32_t)(sad0 + 2 * lambda) << 11) | (uint32_t)(16 * 32 + 16);   // ... and it must not cost more than the zero vector
  if (sadc <= ME_PRED_SAD_FACTOR * ME_EARLY_SAD_PER_LAMBDA * lambda && kc < kmin && kc <= key0) { best = kc; return true; }
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

// an anchor's vector for the rest of its group: one 8-byte store, tag and vector together
__device__ __forceinline__ void publish_anchor(const FrameCtx& f, int mb, int sad_int, int mvx, int mvy) {
  f.me_pub[mb] = ((unsigned long long)((uint32_t)f.pic + 1u) << 32) | (sad_int >= ME_REFINE_MAX_SAD ? 0x10000u : 0u) | (uint32_t)((mvx & 0xff) << 8) | (uint32_t)(mvy & 0xff);
}

// chroma prediction, residual, reconstruction and the macroblock's record; the luma prediction is already in t.pred_y.
// uv_coloc: this lane's word of the co-located chroma reference.
__device__ __forceinline__ void finish_mb(const FrameCtx& f, MbTile& t, int lane, const MbPos& p, int qp, int ylo, int yhi, int mvx, int mvy, uint32_t uv_coloc) {
  const size_t ysz = (size_t)f.cw * f.ch;
  const uint8_t* __restrict__ ref_uv = f.ref + ysz;
  const int r8 = lane >> 1, c8 = (lane & 1) * 8, rc4 = lane >> 2, cc4 = (lane & 3) * 4;
  const int mb = p.mb, mbx = p.mbx, mby = p.mby;
  {
    // chroma: mvC = luma mv, in 1/8 chroma samples (8.4.1.4, 8.4.2.2.2)
    const int xi = mvx >> 3, yi = mvy >> 3, xf = mvx & 7, yf = mvy & 7;
    const int cwc = f.cw >> 1;
    const int ya = clip3i(ylo >> 1, yhi >> 1, mby * 8 + yi + rc4), yb = clip3i(ylo >> 1, yhi >> 1, mby * 8 + yi + rc4 + 1);
    uint32_t out = 0;
    if ((mvx | mvy) == 0) out = uv_coloc;      // zero vector: the co-located pairs, loaded with the first batch
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
  // spills inside it at k_inter_lean's 64 registers
  const uint32_t mv = (uint32_t)(mvx & 0xffff) | ((uint32_t)mvy << 16);
  int luma_bits, chroma_bits;
  int cbp = transform_mb<false>(t, lane, qp, f.coef + (size_t)mb * COEF_BLOCKS * 16, f.nnz + (size_t)mb * 32, luma_bits, chroma_bits);
  if (48 + luma_bits + chroma_bits > MB_BITS_LIMIT) { apply_pcm(t, lane, f.nnz + (size_t)mb * 32); cbp = -1; }   // A.3.1: send raw
  __syncwarp();
  {
    const int ry = mb / f.mbw, rx0 = (mb - ry * f.mbw) * 16;
    const uint2 v = *reinterpret_cast<const uint2*>(&t.rec_y[r8][c8]);
    *reinterpret_cast<uint2*>(f.recon + (size_t)(ry * 16 + r8) * f.cw + rx0 + c8) = v;
    if (lane < 16) {
      const uint2 w = *reinterpret_cast<const uint2*>(&t.rec_uv[r8][c8]);
      *reinterpret_cast<uint2*>(f.recon + ysz + (size_t)(ry * 8 + r8) * f.cw + rx0 + c8) = w;
    }
    if (lane == 0) {
      MbInfo mi; mi.mvx = (int16_t)(mv & 0xffff); mi.mvy = (int16_t)(mv >> 16); mi.type = MB_P16; mi.i16_mode = 0; mi.chroma_mode = 0; mi.cbp = (uint8_t)cbp;
      if (cbp < 0) { mi.mvx = 0; mi.mvy = 0; mi.type = MB_PCM; mi.cbp = 0; }   // too big for CAVLC: I_PCM (transform_mb)
      f.mbinfo[mb] = mi;
    }
  }
}

// Pass A: one warp per macroblock, raster order.  The macroblocks that leave motion estimation through the zero vector or through
// a temporal-predictor hit that needs no refinement are finished here; every other one goes into a queue for k_inter_search —
// anchors into the anchor queue, the rest into the other.  No search and no 48 x 48 window: the registers and shared memory of
// the search do not cap the occupancy of the common case.
__global__ void __launch_bounds__(32 * WARPS_PER_BLOCK, 8) k_inter_lean(FrameCtx f) {
  __shared__ __align__(16) LeanSm sm_all[WARPS_PER_BLOCK];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int mbs = f.mbw * f.mbh;
  const int m = blockIdx.x * WARPS_PER_BLOCK + warp;
  if (m >= mbs) return;
  const MbPos p = mb_pos(f, m);
  LeanSm& sm = sm_all[warp];
  MbTile& t = sm.t;
  const int qp = frame_qp(f), lambda = me_lambda[qp];
  const int ylo = p.band_r0 * 16, yhi = min(f.mbh, p.band_r0 + f.band_rows) * 16 - 1;
  const uint8_t* __restrict__ ref_y = f.ref;
  const int x0 = p.mbx * 16, y0 = p.mby * 16, r8 = lane >> 1, c8 = (lane & 1) * 8;
  // one batch of independent global loads: co-located chroma and luma reference, the previous picture's record, the source block
  const uint32_t uv_coloc = __ldg(reinterpret_cast<const uint32_t*>(f.ref + (size_t)f.cw * f.ch + (size_t)(p.mby * 8 + (lane >> 2)) * f.cw + x0 + (lane & 3) * 4));
  const uint2 z = __ldg(reinterpret_cast<const uint2*>(ref_y + (size_t)(y0 + r8) * f.cw + x0 + c8));
  const MbInfo prev = f.mbinfo_prev[m];
  const uint2 c = stage_source(f, t, lane, x0, p.mby);
  __syncwarp();

  // zero-motion early termination: co-located block within the quantisation noise of this QP
  const int sad0 = __reduce_add_sync(FULL, (int)sad4acc(c.x, z.x, sad4acc(c.y, z.y, 0u)));
  int mvx = 0, mvy = 0, sad_int = 0;
  if (sad0 <= ME_EARLY_SAD_PER_LAMBDA * lambda) {
    *reinterpret_cast<uint2*>(&t.pred_y[r8][c8]) = z;
  } else {
    // the temporal predictor, with the 24 rows x 8 words around it that its test and its prediction touch (k_inter_search stages
    // the same words at the same window coordinates).  A picture-edge macroblock, which needs per-sample clamping, is deferred.
    const int cdx = (prev.mvx + 2) >> 2, cdy = (prev.mvy + 2) >> 2;
    const bool try_pred = prev.type == MB_P16 && cdx >= -15 && cdx <= 14 && cdy >= -15 && cdy <= 15;
    bool hit = false;
    if (try_pred && x0 >= 16 && x0 + 32 <= f.cw) {
      const int ra = min(max(13 + cdy, 0), WIN_ROWS - PW_ROWS), wa = min(max((13 + cdx) >> 2, 0), WIN_WORDS - PW_WORDS);
      const uint32_t* base = reinterpret_cast<const uint32_t*>(ref_y + x0 - 16);
      uint32_t v[6];
#pragma unroll
      for (int k = 0; k < 6; k++) {
        const int idx = lane + 32 * k;
        v[k] = __ldg(base + (size_t)clip3i(ylo, yhi, y0 - 16 + ra + (idx >> 3)) * (f.cw >> 2) + wa + (idx & 7));
      }
#pragma unroll
      for (int k = 0; k < 6; k++) sm.pw[(lane + 32 * k) >> 3][lane & 7] = v[k];
      __syncwarp();
      const WinView w{&sm.pw[0][0], PW_WORDS, ra, wa};
      uint32_t best;
      // a hit whose previous vector was fractional is refined: k_inter_search does that
      hit = test_candidate(w, t, lane, cdx, cdy, lambda, sad0, best) && ((prev.mvx | prev.mvy) & 3) == 0;
      if (hit) {
        full_sample_pred(w, t, lane, 16 + cdx, 16 + cdy);
        mvx = 4 * cdx; mvy = 4 * cdy;
        sad_int = (int)(best >> 11) - lambda * (se_bits_dev(mvx) + se_bits_dev(mvy));
      }
    }
    if (!hit) {
      if (lane == 0) {
        const int qi = p.anchor ? 0 : 1;
        f.me_queue[2 + qi * mbs + atomicAdd(&f.me_queue[qi], 1)] = m;
      }
      return;
    }
  }
  if (p.anchor && lane == 0) publish_anchor(f, m, sad_int, mvx, mvy);
  finish_mb(f, t, lane, p, qp, ylo, yhi, mvx, mvy, uv_coloc);
}

// One macroblock that k_inter_lean queued, from the start: its zero-motion and temporal-predictor tests are repeated on the same
// inputs (source, reference and the previous picture's records are not written during the analysis of a picture) and so fail, or
// hit, exactly as they did there.
__device__ __forceinline__ void search_mb(const FrameCtx& f, InterSm& sm, int lane, const MbPos& p) {
  const int mb = p.mb, mbx = p.mbx, mby = p.mby, x0 = mbx * 16, y0 = mby * 16;
  const bool anchor = p.anchor;
  MbTile& t = sm.t;
  const WinView win{&sm.win[0][0], WIN_WORDS, 0, 0};
  const int qp = frame_qp(f);
  // reference rows this macroblock may touch: its own band (the band's decoder pads at the band's edges, 8.4.2.2.1)
  const int ylo = p.band_r0 * 16, yhi = min(f.mbh, p.band_r0 + f.band_rows) * 16 - 1;
  const size_t ysz = (size_t)f.cw * f.ch;
  const uint8_t* __restrict__ ref_y = f.ref; const uint8_t* __restrict__ ref_uv = f.ref + ysz;
  const int r8 = lane >> 1, c8 = (lane & 1) * 8, rc4 = lane >> 2, cc4 = (lane & 3) * 4;

  // ---- stage the source block and the search window ------------------------------------------------
  // one batch of independent global loads: source block, co-located reference block, and — speculatively, they are needed again a
  // dependent-load latency later otherwise — the co-located chroma reference (the chroma prediction of a zero vector) and this
  // macroblock's record of the previous picture (temporal predictor)
  const uint32_t uv_coloc = __ldg(reinterpret_cast<const uint32_t*>(ref_uv + (size_t)(mby * 8 + rc4) * f.cw + x0 + cc4));
  const MbInfo prev = f.mbinfo_prev[mb];                    // the previous picture's record (other half of the double buffer)
  {
    stage_source(f, t, lane, x0, mby);
    // the co-located 16x16 block first (window rows 16..31, words 4..7)
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const int i = lane + 32 * k;
      sm.win[16 + (i >> 2)][4 + (i & 3)] = __ldg(reinterpret_cast<const uint32_t*>(ref_y + (size_t)(y0 + (i >> 2)) * f.cw + x0) + (i & 3));
    }
  }
  __syncwarp();

  // ---- zero-motion early termination (DESIGN.md §5.3): co-located block within the quantisation noise of this QP ----
  const int lambda = me_lambda[qp];
  uint32_t best = (uint32_t)(16 * 32 + 16);      // candidate (0,0)
  int sad0;
  {
    const uint32_t* w0p = &sm.win[16 + r8][4 + (c8 >> 2)];
    const uint32_t s0 = sad4acc(*reinterpret_cast<const uint32_t*>(&t.cur_y[r8][c8]), w0p[0],
                                sad4acc(*reinterpret_cast<const uint32_t*>(&t.cur_y[r8][c8 + 4]), w0p[1], 0u));
    sad0 = __reduce_add_sync(FULL, (int)s0);
    if (sad0 > ME_EARLY_SAD_PER_LAMBDA * lambda) best = 0xffffffffu;
  }
  // ---- not static: stage the reference.  A macroblock that carries a vector from the previous picture first gets only what the
  // temporal-predictor test, the refinement around it and the final prediction can touch — 24 rows x 8 words around the predicted
  // position instead of the 48 x 12 window; the rest follows only if the predictor is rejected and the search has to run.
  const int cdx = (prev.mvx + 2) >> 2, cdy = (prev.mvy + 2) >> 2;
  const bool try_pred = prev.type == MB_P16 && cdx >= -15 && cdx <= 14 && cdy >= -15 && cdy <= 15;     // the zero vector included
  const bool x_inside = x0 >= 16 && x0 + 32 <= f.cw;
  bool window_complete = false;
  auto stage_window = [&]() {
    if (x_inside) {   // 512 more words: lanes 0..23 take (row pair j, word) = two rows of 12 words per step — no index arithmetic
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
  if (best == 0xffffffffu) {
    if (x_inside && try_pred) {
      // rows [13+cdy, 36+cdy] and bytes [13+cdx, 34+cdx] of the window cover the 3x3 predictor test (rows 15+cdy..32+cdy), the 6-tap
      // support of a refinement around it (-3..+18) and the prediction; clamped so that 24 rows x 8 words stay inside the window
      const int ra = min(max(13 + cdy, 0), WIN_ROWS - PW_ROWS), wa = min(max((13 + cdx) >> 2, 0), WIN_WORDS - PW_WORDS);
      const uint32_t* base = reinterpret_cast<const uint32_t*>(ref_y + x0 - 16);
      uint32_t v[6];
#pragma unroll
      for (int k = 0; k < 6; k++) {
        const int idx = lane + 32 * k, row = ra + (idx >> 3), w = wa + (idx & 7);
        v[k] = __ldg(base + (size_t)clip3i(ylo, yhi, y0 - 16 + row) * (f.cw >> 2) + w);
      }
#pragma unroll
      for (int k = 0; k < 6; k++) {
        const int idx = lane + 32 * k;
        sm.win[ra + (idx >> 3)][wa + (idx & 7)] = v[k];
      }
      __syncwarp();
    } else stage_window();
  }
  // ---- temporal predictor: the vector this macroblock had in the previous picture, rounded to full samples (scrolling / panning
  // content repeats it; the zero vector counts: static content whose co-located SAD sits just above the early-termination threshold
  // would otherwise search only to find (0,0) again); quarter-sample refinement then runs as after a search. ----
  bool pred_hit = false, pred_frac = false, reduced = false;
  if (best == 0xffffffffu && try_pred && test_candidate(win, t, lane, cdx, cdy, lambda, sad0, best)) { pred_hit = true; pred_frac = ((prev.mvx | prev.mvy) & 3) != 0; }
  // ---- anchor predictor (oracle/h264_ref.c encode_inter_mb): the temporal predictor failed (or there was none) — motion that
  // STARTS in this picture.  Instead of one exhaustive search per macroblock, try what this group's anchor has found. ----
  if (best == 0xffffffffu && !anchor) {
    if (!window_complete) stage_window();       // any candidate position may be tried; needed by the search anyway if it is rejected
    // written by k_inter_lean or by the anchor pass, both earlier in stream order.  The tag is always there; were it missing, the
    // macroblock would run the exhaustive search and the stream would differ from the oracle's.
    const unsigned long long v = f.me_pub[(size_t)p.ay * f.mbw + p.ax];
    const bool have = (uint32_t)(v >> 32) == (uint32_t)f.pic + 1u;
    const int amvx = (int)(int8_t)(v >> 8), amvy = (int)(int8_t)v;
    const int kx = (amvx + 2) >> 2, ky = (amvy + 2) >> 2;
    const bool zero_again = (kx | ky) == 0 && try_pred && (cdx | cdy) == 0;      // the zero vector is not tested twice
    if (have && !zero_again && kx >= -15 && kx <= 14 && ky >= -15 && ky <= 15 && test_candidate(win, t, lane, kx, ky, lambda, sad0, best)) { pred_hit = true; pred_frac = ((amvx | amvy) & 3) != 0; }
    // new content: the anchor's exhaustive search found nothing (bit 16) and the co-located block is as far off — the search
    // shrinks to the rows around dy = 0: picking the least bad of 1089 noise candidates buys hardly more than picking it of 160
    else reduced = have && ((v >> 16) & 1) != 0 && sad0 >= ME_REFINE_MAX_SAD;
  }
  const bool searched = best == 0xffffffffu;
  if (searched && !window_complete) stage_window();          // predictor rejected: the search needs the whole window
  if (searched) best = reduced ? search_rows<ME_NEWCONTENT_DY>(sm, lane, lambda) : search_rows<16>(sm, lane, lambda);
  const int dyi = (best & 2047) >> 5, dxi = best & 31, dx = dxi - 16, dy = dyi - 16;

  // ---- quarter-sample refinement (DESIGN.md §5.3; oracle/h264_ref.c encode_inter_mb) ---------------------------------
  int mvx = 4 * dx, mvy = 4 * dy;
  // refine only inside the window (6-tap support [-3,+18]) and when the full-sample match is not already within the
  // quantisation noise of this QP (same threshold as the zero-motion early termination)
  const int sad_int = (searched || pred_hit) ? (int)(best >> 11) - lambda * (se_bits_dev(4 * dx) + se_bits_dev(4 * dy)) : 0;
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
        const uint32_t cost = (uint32_t)(sad + lambda * (se_bits_dev(4 * dx + qx) + se_bits_dev(4 * dy + qy) + (((qx | qy) & 3) ? ME_FRAC_PENALTY_BITS : 0)));
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
  if (anchor && lane == 0) publish_anchor(f, mb, sad_int, mvx, mvy);
  if (!refine) full_sample_pred(win, t, lane, dxi, dyi);
  finish_mb(f, t, lane, p, qp, ylo, yhi, mvx, mvy, uv_coloc);
}

// Passes B and C: the queue k_inter_lean filled (0: anchors, 1: the rest), walked by a grid of the kernel's resident capacity.  No
// decision here depends on another entry of the same queue, so the order inside a queue does not matter.
__global__ void __launch_bounds__(32 * WARPS_PER_BLOCK, 5) k_inter_search(FrameCtx f, int queue) {
  __shared__ __align__(16) InterSm sm_all[WARPS_PER_BLOCK];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = f.me_queue[queue];
  const int* q = f.me_queue + 2 + (size_t)queue * f.mbw * f.mbh;
  for (int i = blockIdx.x * WARPS_PER_BLOCK + warp; i < n; i += gridDim.x * WARPS_PER_BLOCK) {
    search_mb(f, sm_all[warp], lane, mb_pos(f, q[i]));
    __syncwarp();
  }
}

cudaError_t inter_search_grid(int* blocks) {
  int dev = 0, sms = 0, per_sm = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_inter_search, 32 * WARPS_PER_BLOCK, 0);
  *blocks = sms * per_sm;
  return e;
}

int launch_inter(const FrameCtx& f, cudaStream_t st) {
  // both queues empty; the counters are only read by the two k_inter_search launches that follow
  cudaMemsetAsync(f.me_queue, 0, 2 * sizeof(int), st);
  k_inter_lean<<<(f.mbw * f.mbh + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, 32 * WARPS_PER_BLOCK, 0, st>>>(f);
  k_inter_search<<<f.search_blocks, 32 * WARPS_PER_BLOCK, 0, st>>>(f, 0);   // anchors
  k_inter_search<<<f.search_blocks, 32 * WARPS_PER_BLOCK, 0, st>>>(f, 1);   // the rest: read the anchors' vectors
  return 3;
}

}  // namespace b2v
