// h264_intra.cu — IDR pictures: Intra4x4 / Intra16x16 macroblocks (ITU-T H.264 8.3.1, 8.3.3 luma; 8.3.4 chroma).
//
// One block of THREE warps per slice.  IDR slices never span rows (a grid of 1 x slice_cols macroblocks, DESIGN.md §5.2), so
// no macroblock has a neighbour above and no block depends on another.  Inside a slice intra prediction needs the reconstructed
// left neighbour, so its macroblocks are a serial chain.  The chain is latency-bound (one dependent shuffle / shared-memory round
// trip after the other), so the two ways of coding a macroblock run side by side: warp 0 codes Intra16x16 + chroma while
// warps 1 and 2 run the Intra4x4 pass.
//
// Per macroblock the luma is coded BOTH ways and the better one kept:
//   Intra4x4   16 blocks in decoding order; per block the 32 lanes evaluate 8 modes x 4 rows (+ horizontal-up)
//              in parallel, key = (SAD + lambda*(mode == predicted ? 1 : 4))*16 + mode, then lanes 0..15 hold one
//              residual sample each and run the 4x4 transform / quantisation / reconstruction with warp shuffles
//   Intra16x16 luma mode = argmin(SAD*4 + mode); transform_mb<true> (one lane per 4x4 block, DC Hadamard)
//   decision   J = SSD + rd_lambda(qp) * luma bits (exact CAVLC size with the longest coeff_token); smaller J wins.
// Chroma: mode = argmin((SAD Cb + SAD Cr)*4 + mode).  Encoder decisions: DESIGN.md §5.2; CPU restatement:
// oracle/h264_ref.c encode_intra_mb(), intra4x4_pass().
#include "h264_common.cuh"
#include "h264_kernels.h"

namespace b2v {

constexpr int I4_SKIP_SAD_PER_LAMBDA = 32;   // Intra4x4 is only tried when the best Intra16x16 SAD exceeds 32*lambda

__device__ __forceinline__ uint32_t rep4(int v) { return (uint32_t)v * 0x01010101u; }

struct IntraNb {                             // what a macroblock takes from its left neighbour (it has none above)
  uint8_t left_y[16];
  uint8_t left_uv[16];                       // interleaved Cb,Cr: [y*2+c]
  int cdc[8];                                // chroma DC prediction per (comp*4 + blk)
  uint8_t left_modes[4];                     // Intra4x4PredMode of the left macroblock's right column (2 if it is not I4x4)
};

struct I4State {
  alignas(16) int16_t lv[16][16];            // [blkIdx][scan position]; read back with 16-byte loads
  alignas(16) uint8_t code[9][16];           // shared-memory copy of i4_pred_code (read as 32-bit words)
  alignas(16) uint8_t v[2][64];              // per Intra4x4 warp: X | F2 | F3 | DC of its current block (see i4_pred_code)
  int mode_bits_part;                        // mode bits accumulated by the second Intra4x4 warp
  uint8_t rt[17][24];                        // framed reconstruction (see the Intra4x4 pass)
  uint8_t nnz[16];                           // raster block position
  uint8_t modes[16];                         // raster block position
};

__device__ __forceinline__ int f3(int a, int b, int c) { return (a + 2 * b + c + 2) >> 2; }
__device__ __forceinline__ int f2(int a, int b) { return (a + b + 1) >> 1; }

// Intra4x4 prediction as a table lookup (8.3.1.2.1-9).  The 13 neighbouring samples are laid out as
//   X[0] = l3 (dup), X[1..4] = l3 l2 l1 l0, X[5] = M (above-left), X[6..13] = t0..t7, X[14] = t7 (dup)
// and every predicted sample of every mode is one of: X[i] (code i), F2[i] = (X[i]+X[i+1]+1)>>1 (code 16+i),
// F3[i] = (X[i-1]+2X[i]+X[i+1]+2)>>2 (code 32+i) or the DC value (code 48).  One shared-memory array V[64] holds all
// of them, so the nine modes are evaluated without any divergent control flow.  (Generated from the formulas of the
// Recommendation and checked against them exhaustively; the CPU oracle evaluates the formulas directly.)
__device__ const uint8_t i4_pred_code[9][16] = {
  { 6, 7, 8, 9, 6, 7, 8, 9, 6, 7, 8, 9, 6, 7, 8, 9 },                     // 0 vertical
  { 4, 4, 4, 4, 3, 3, 3, 3, 2, 2, 2, 2, 1, 1, 1, 1 },                     // 1 horizontal
  { 48, 48, 48, 48, 48, 48, 48, 48, 48, 48, 48, 48, 48, 48, 48, 48 },     // 2 DC
  { 39, 40, 41, 42, 40, 41, 42, 43, 41, 42, 43, 44, 42, 43, 44, 45 },     // 3 diagonal down-left
  { 37, 38, 39, 40, 36, 37, 38, 39, 35, 36, 37, 38, 34, 35, 36, 37 },     // 4 diagonal down-right
  { 21, 22, 23, 24, 37, 38, 39, 40, 36, 21, 22, 23, 35, 37, 38, 39 },     // 5 vertical-right
  { 20, 37, 38, 39, 19, 36, 20, 37, 18, 35, 19, 36, 17, 34, 18, 35 },     // 6 horizontal-down
  { 22, 23, 24, 25, 39, 40, 41, 42, 23, 24, 25, 26, 40, 41, 42, 43 },     // 7 vertical-left
  { 19, 35, 18, 34, 18, 34, 17, 33, 17, 33, 1, 1, 1, 1, 1, 1 },           // 8 horizontal-up
};
__device__ __forceinline__ bool i4_mode_ok(int mode, bool has_a, bool has_b, bool has_d) {
  switch (mode) {
    case 0: case 3: case 7: return has_b;
    case 1: case 8: return has_a;
    case 2: return true;
    default: return has_a && has_b && has_d;
  }
}
// (above-right availability and the inverse zig-zag are packed literals in the kernel: the above-right samples of a block
//  are available when they lie inside the macroblock, raster { 0,0,0,0, 1,0,1,0, 1,1,1,0, 1,0,1,0 } = bit mask 0x5750)

// one 1-D stage of the forward / inverse core transform for the element `k` of (a,b,c,d)
__device__ __forceinline__ int fwd1(int k, int a, int b, int c, int d) {
  return k == 0 ? a + b + c + d : k == 1 ? 2 * (a - d) + (b - c) : k == 2 ? (a + d) - (b + c) : (a - d) - 2 * (b - c);
}
__device__ __forceinline__ int inv1(int k, int p0, int p1, int p2, int p3) {
  const int e0 = p0 + p2, e1 = p0 - p2, e2 = (p1 >> 1) - p3, e3 = p1 + (p3 >> 1);
  return k == 0 ? e0 + e3 : k == 1 ? e1 + e2 : k == 2 ? e1 - e2 : e0 - e3;
}

// Intra16x16 luma mode decision (8.3.3) without a neighbour above: horizontal (needs the left one) or DC, key = SAD*4 + mode;
// p = the value of this lane's 8 predicted samples, 4 to a word (both modes repeat one value along a row)
struct I16Dec { int key, mode; uint32_t p; };
__device__ __forceinline__ I16Dec i16_decide(const IntraNb& nb, const MbTile& t, int lane, bool has_left) {
  const int r8 = lane >> 1, c8 = (lane & 1) * 8;
  const uint32_t cy0 = *reinterpret_cast<const uint32_t*>(&t.cur_y[r8][c8]);
  const uint32_t cy1 = *reinterpret_cast<const uint32_t*>(&t.cur_y[r8][c8 + 4]);
  int sum_l = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) sum_l += nb.left_y[i];
  const uint32_t ph = rep4(nb.left_y[r8]), pd = rep4(has_left ? (sum_l + 8) >> 4 : 128);
  int best_key = 0x7fffffff, best_mode = 2, s;
  if (has_left) { s = __reduce_add_sync(FULL, __vsadu4(cy0, ph) + __vsadu4(cy1, ph)); if (s * 4 + 1 < best_key) { best_key = s * 4 + 1; best_mode = 1; } }
  s = __reduce_add_sync(FULL, __vsadu4(cy0, pd) + __vsadu4(cy1, pd)); if (s * 4 + 2 < best_key) { best_key = s * 4 + 2; best_mode = 2; }
  I16Dec d;
  d.key = best_key; d.mode = best_mode;
  d.p = best_mode == 1 ? ph : pd;
  return d;
}

// what the Intra4x4 warp hands to the deciding warp
struct I4Result { int tried, mode_bits, cbp, bits; long long d; };

__device__ __forceinline__ void i4_pair_barrier() { asm volatile("bar.sync 1, 64;" ::: "memory"); }   // the two Intra4x4 warps

// CUT (B2V_FLAG_SCENE_CUT): a P picture, launched behind k_scene_cut on the IDR grid; it codes the picture only when it was cut, at the
// P picture's QP (f.idr is 0), over what the P analysis wrote.
template <bool CUT>
__global__ void __launch_bounds__(96) k_intra_rows(FrameCtx f) {
  __shared__ __align__(16) MbTile t;
  __shared__ __align__(16) IntraNb nb;
  __shared__ __align__(16) I4State i4;
  __shared__ I4Result r4;
  if (CUT && !f.scut->cut[f.pic & 1]) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const SliceGeo geo = slice_geo(f, blockIdx.x);        // columns [x0, x1) of row row0
  const int mby = geo.row0;
  const int qp = frame_qp(f);
  const int lambda = me_lambda[qp];
  const size_t ysz = (size_t)f.cw * f.ch;
  const int r8 = lane >> 1, c8 = (lane & 1) * 8;            // this lane's 8 luma pixels
  const int rc4 = lane >> 2, cc4 = (lane & 3) * 4;          // this lane's 4 interleaved chroma bytes
  const QuantParams q4 = make_quant(qp, true);
  // lane-invariant roles inside the Intra4x4 pass
  const int px = lane & 3, py = (lane >> 2) & 3, rpos = py * 4 + px, rowb = lane & ~3, colb = (lane & 16) | px;
  const int cls = pos_class(rpos), mf_l = q4.mf[cls], dq_l = q4.dq[cls];
  const int izz = (int)((0xFEA9DB83C7426510ull >> (4 * rpos)) & 15ull);      // raster -> scan position (inverse zig-zag), nibble-packed
  const int lm = lane >> 2, ly = lane & 3;                                    // candidate mode / row evaluated by this lane
  const int lm_need = (lm == 0 || lm == 3 || lm == 7) ? 0 : lm == 1 ? 1 : lm == 2 ? 2 : 3;   // needs: above / left / nothing / all three
  if (threadIdx.x < 4) nb.left_modes[threadIdx.x] = 2;
  for (int i = threadIdx.x; i < 144; i += 96) (&i4.code[0][0])[i] = (&i4_pred_code[0][0])[i];
  __syncthreads();
  const uint32_t cm = *reinterpret_cast<const uint32_t*>(&i4.code[lm][ly * 4]);   // V-indices of this lane's four predicted samples
  const uint32_t ch = *reinterpret_cast<const uint32_t*>(&i4.code[8][ly * 4]);    // ... for horizontal-up

  for (int mbx = geo.x0; mbx < geo.x1; mbx++) {
    const int mb = mby * f.mbw + mbx;
    const bool has_left = mbx > geo.x0;
    if (warp == 0) stage_source(f, t, lane, mbx * 16, mby, ysz);     // load the current macroblock
    __syncthreads();
    int best_mode = 2, cbest = 0, cbp = 0, luma_bits16 = 0, chroma_bits = 0;
    long long d16 = 0;
    int16_t* coef_mb = f.coef + (size_t)mb * COEF_BLOCKS * 16;
    uint8_t* nnz_mb = f.nnz + (size_t)mb * 32;
    if (warp == 0) {
    // ================= warp 0: Intra16x16 luma + chroma ==================================================
    // chroma DC predictors (8.3.4.1-3), one (component, block) per lane 0..7
    if (lane < 8) {
      const int c = lane >> 2, by = ((lane & 3) >> 1) * 4;
      int sl = 0;
#pragma unroll
      for (int i = 0; i < 4; i++) sl += nb.left_uv[(by + i) * 2 + c];
      nb.cdc[lane] = has_left ? (sl + 2) >> 2 : 128;
    }
    {
      const I16Dec d = i16_decide(nb, t, lane, has_left);
      best_mode = d.mode;
      *reinterpret_cast<uint32_t*>(&t.pred_y[r8][c8]) = d.p;
      *reinterpret_cast<uint32_t*>(&t.pred_y[r8][c8 + 4]) = d.p;
    }
    __syncwarp();   // nb.cdc visible
    // ---- chroma mode decision: DC or (with a left neighbour) horizontal, key = (SAD Cb + SAD Cr)*4 + mode -----
    const uint32_t cc = *reinterpret_cast<const uint32_t*>(&t.cur_uv[rc4][cc4]);   // Cb0 Cr0 Cb1 Cr1 at x = (lane&3)*2, +1
    uint32_t qd, qh;
    {
      const int blk = (rc4 >> 2) * 2 + ((lane & 3) >> 1);
      qd = (uint32_t)nb.cdc[blk] | ((uint32_t)nb.cdc[4 + blk] << 8);
      qd |= qd << 16;
      qh = (uint32_t)nb.left_uv[rc4 * 2] | ((uint32_t)nb.left_uv[rc4 * 2 + 1] << 8);
      qh |= qh << 16;
    }
    int cbest_key = 0x7fffffff;
    cbest = 0;
    {
      int s = __reduce_add_sync(FULL, __vsadu4(cc, qd)); if (s * 4 + 0 < cbest_key) { cbest_key = s * 4 + 0; cbest = 0; }
      if (has_left) { s = __reduce_add_sync(FULL, __vsadu4(cc, qh)); if (s * 4 + 1 < cbest_key) { cbest_key = s * 4 + 1; cbest = 1; } }
    }
    *reinterpret_cast<uint32_t*>(&t.pred_uv[rc4][cc4]) = cbest == 0 ? qd : qh;
    __syncwarp();

    // ---- Intra16x16 coding (also codes the chroma, which is identical either way) --------------------------
    cbp = transform_mb<true>(t, lane, qp, coef_mb, nnz_mb, luma_bits16, chroma_bits);
    __syncwarp();
    {
      int s = 0;
#pragma unroll
      for (int j = 0; j < 8; j++) { const int e = (int)t.cur_y[r8][c8 + j] - (int)t.rec_y[r8][c8 + j]; s += e * e; }
      d16 = __reduce_add_sync(FULL, s);
    }
    } else {
    // ================= warps 1 and 2: Intra4x4 candidate ====================================================
    // The 16 blocks form a wavefront (a block needs its left, above, above-left and above-right neighbours): at step
    // T = bx + 2*by at most two blocks are ready, so the pair of warps finishes the macroblock in 10 steps instead of 16.
    const int u = warp - 1;
    uint8_t* const V = i4.v[u];
    const int best_key = i16_decide(nb, t, lane, has_left).key;      // same decision as warp 0 (reads only)
    // ---- Intra4x4 candidate: 16 blocks in decoding order ----------------------------------------------
    // rt = reconstruction with a one-sample frame: rt[y+1][x+1] is macroblock sample (x,y), column 0 holds the neighbours to the
    // left.  Row 0 stands for the samples above the macroblock, which are not available: no mode that reads them is selected.
    const bool try_i4 = (best_key >> 2) > I4_SKIP_SAD_PER_LAMBDA * lambda;      // nearly flat macroblocks go straight to Intra16x16
    int mode_bits4 = 0, cbp4 = 0, bits4_cavlc = 0;
    long long d4 = 0;
    if (try_i4) {
      if (u == 0 && lane < 16) i4.rt[1 + lane][0] = nb.left_y[lane];
      i4_pair_barrier();
      for (int T = 0; T < 10; T++) {
        // raster position of this warp's block at step T (nibble-packed): warp u=0 takes row 0 and columns 2,3; u=1 columns 0,1 of rows 1..3
        const int rp = u == 0 ? (int)((0xFEBA763210ull >> (4 * T)) & 15ull) : (T >= 2 && T <= 7 ? (int)((0xDC985400u >> (4 * T)) & 15u) : -1);
        if (rp >= 0) {
        const int bx = rp & 3, by = rp >> 2;
        const int blk = (by >> 1) * 8 + (bx >> 1) * 4 + (by & 1) * 2 + (bx & 1);          // blkIdx in decoding order
        const bool has_a = bx > 0 || has_left, has_b = by > 0, has_d = by > 0 && (bx > 0 || has_left);
        const bool has_c = (0x5750u >> rp) & 1u;       // above-right samples inside the macroblock
        if (lane < 15) {        // X[lane]: neighbouring samples of this block (values of unavailable ones are never selected)
          int row = by * 4, col = bx * 4;
          if (lane < 5) row += (lane == 0 ? 3 : 4 - lane) + 1;
          else if (lane > 5) { int j = lane == 14 ? 7 : lane - 6; if (j >= 4 && !has_c) j = 3; col += 1 + j; }   // 8.3.1.2: repeat p[3,-1]
          V[lane] = i4.rt[row][col];
        }
        __syncwarp();
        if (lane < 14) V[16 + lane] = (uint8_t)f2(V[lane], V[lane + 1]);
        else if (lane >= 16 && lane < 29) { const int i = lane - 15; V[32 + i] = (uint8_t)f3(V[i - 1], V[i], V[i + 1]); }
        else if (lane == 31) {
          const int st = V[6] + V[7] + V[8] + V[9], sl = V[1] + V[2] + V[3] + V[4];
          V[48] = (uint8_t)(has_a && has_b ? (st + sl + 4) >> 3 : has_b ? (st + 2) >> 2 : has_a ? (sl + 2) >> 2 : 128);
        }
        __syncwarp();
        // predicted mode (8.3.1.1): 2 when the block to the left or above is not available, which is always so in the top row
        int pm = 2;
        if (by > 0) {
          const int ma = bx > 0 ? (int)i4.modes[by * 4 + bx - 1] : has_left ? (int)nb.left_modes[by] : -1;
          if (ma >= 0) pm = min(ma, (int)i4.modes[(by - 1) * 4 + bx]);
        }
        // modes 0..7: lane = mode*4 + row; mode 8: every group of four lanes evaluates it as well
        const uint32_t crow = *reinterpret_cast<const uint32_t*>(&t.cur_y[by * 4 + ly][bx * 4]);
        const uint32_t pm4 = (uint32_t)V[cm & 255] | ((uint32_t)V[(cm >> 8) & 255] << 8) | ((uint32_t)V[(cm >> 16) & 255] << 16) | ((uint32_t)V[cm >> 24] << 24);
        const uint32_t p84 = (uint32_t)V[ch & 255] | ((uint32_t)V[(ch >> 8) & 255] << 8) | ((uint32_t)V[(ch >> 16) & 255] << 16) | ((uint32_t)V[ch >> 24] << 24);
        int sad_m = (int)__vsadu4(crow, pm4), sad_hu = (int)__vsadu4(crow, p84);
        sad_m += __shfl_xor_sync(FULL, sad_m, 1); sad_hu += __shfl_xor_sync(FULL, sad_hu, 1);
        sad_m += __shfl_xor_sync(FULL, sad_m, 2); sad_hu += __shfl_xor_sync(FULL, sad_hu, 2);
        const bool ok_m = lm_need == 0 ? has_b : lm_need == 1 ? has_a : lm_need == 2 ? true : (has_a && has_b && has_d);
        uint32_t key = 0xffffffffu;
        if (ok_m) key = (uint32_t)((sad_m + lambda * (lm == pm ? 1 : 4)) * 16 + lm);
        if (has_a) key = min(key, (uint32_t)((sad_hu + lambda * (8 == pm ? 1 : 4)) * 16 + 8));
        key = __reduce_min_sync(FULL, key);
        const int mode = key & 15;
        mode_bits4 += mode == pm ? 1 : 4;
        // lanes 0..15: one sample each; transform / quantise / reconstruct with shuffles (lanes 16..31 mirror 0..15)
        const int pred = V[i4.code[mode][rpos]];
        const int res = (int)t.cur_y[by * 4 + py][bx * 4 + px] - pred;
        int v = fwd1(px, __shfl_sync(FULL, res, rowb), __shfl_sync(FULL, res, rowb + 1), __shfl_sync(FULL, res, rowb + 2), __shfl_sync(FULL, res, rowb + 3));
        v = fwd1(py, __shfl_sync(FULL, v, colb), __shfl_sync(FULL, v, colb + 4), __shfl_sync(FULL, v, colb + 8), __shfl_sync(FULL, v, colb + 12));
        const int level = quant1(v, mf_l, q4.f, q4.qbits);
        const unsigned nzm = __ballot_sync(FULL, level != 0) & 0xffffu;
        if (lane < 16) i4.lv[blk][izz] = (int16_t)level;
        int d = (level * dq_l) << q4.qshift;
        d = inv1(px, __shfl_sync(FULL, d, rowb), __shfl_sync(FULL, d, rowb + 1), __shfl_sync(FULL, d, rowb + 2), __shfl_sync(FULL, d, rowb + 3));
        d = inv1(py, __shfl_sync(FULL, d, colb), __shfl_sync(FULL, d, colb + 4), __shfl_sync(FULL, d, colb + 8), __shfl_sync(FULL, d, colb + 12));
        if (lane < 16) i4.rt[by * 4 + py + 1][bx * 4 + px + 1] = (uint8_t)clip255(pred + ((d + 32) >> 6));
        if (lane == 0) { i4.modes[by * 4 + bx] = (uint8_t)mode; i4.nnz[by * 4 + bx] = (uint8_t)__popc(nzm); }
        }
        if (T == 9 && u == 1 && lane == 0) i4.mode_bits_part = mode_bits4;
        i4_pair_barrier();
      }
      if (u == 0) {
      mode_bits4 += i4.mode_bits_part;
      // I4 luma size + distortion
#pragma unroll
      for (int b = 0; b < 16; b++) if (i4.nnz[(((b >> 3) * 2 + ((b >> 1) & 1)) * 4) + ((b >> 2) & 1) * 2 + (b & 1)]) cbp4 |= 1 << (b >> 2);
      {
        CountSink cs;
        if (lane >= 1 && lane <= 16 && ((cbp4 >> ((lane - 1) >> 2)) & 1)) cavlc_block(cs, &i4.lv[lane - 1][0], 16, NC_WORST);
        bits4_cavlc = __reduce_add_sync(FULL, cs.n);
      }
      {
        int sd = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) { const int e = (int)t.cur_y[r8][c8 + j] - (int)i4.rt[r8 + 1][c8 + j + 1]; sd += e * e; }
        d4 = __reduce_add_sync(FULL, sd);
      }
      }
    }
    if (u == 0 && lane == 0) { r4.tried = try_i4; r4.mode_bits = mode_bits4; r4.cbp = cbp4; r4.bits = bits4_cavlc; r4.d = d4; }
    }
    __syncthreads();
    // ================= decision, commit and write-out (warp 0) ============================================
    if (warp == 0) {
    const bool try_i4 = r4.tried != 0;
    const int mode_bits4 = r4.mode_bits, cbp4 = r4.cbp, bits4_cavlc = r4.bits;
    const long long d4 = r4.d;
    const long long l2 = rd_lambda[qp];
    const bool use_i4 = try_i4 && d4 + l2 * (8 + bits4_cavlc + mode_bits4) < d16 + l2 * (8 + luma_bits16);
    int est;
    if (use_i4) {     // commit the 4x4 result over the 16x16 one
#pragma unroll
      for (int j = 0; j < 8; j++) t.rec_y[r8][c8 + j] = i4.rt[r8 + 1][c8 + j + 1];
      if (lane < 16) {
        const uint4* src = reinterpret_cast<const uint4*>(&i4.lv[lane][0]);
        uint4* dst = reinterpret_cast<uint4*>(coef_mb + (1 + lane) * 16);
        dst[0] = src[0]; dst[1] = src[1];
        nnz_mb[lane] = i4.nnz[lane];
        f.i4modes[(size_t)mb * 16 + lane] = i4.modes[lane];
      }
      cbp = cbp4 | (cbp & 0x30);
      est = 96 + bits4_cavlc + chroma_bits;
    } else {
      est = 48 + luma_bits16 + chroma_bits;
    }
    int type = use_i4 ? MB_I4 : MB_I16;
    __syncwarp();
    if (est > MB_BITS_LIMIT) { apply_pcm(t, lane, nnz_mb); type = MB_PCM; cbp = 0; __syncwarp(); }   // A.3.1: send raw
    {
      store_recon(f, t, lane, mbx * 16, mby, ysz);
      // right column becomes the next macroblock's left neighbour
      if (lane < 16) nb.left_y[lane] = t.rec_y[lane][15];
      else nb.left_uv[lane - 16] = t.rec_uv[(lane - 16) >> 1][14 + ((lane - 16) & 1)];
      if (lane < 4) nb.left_modes[lane] = type == MB_I4 ? i4.modes[lane * 4 + 3] : (uint8_t)2;
      if (lane == 0) {
        MbInfo mi; mi.mvx = 0; mi.mvy = 0; mi.type = (uint8_t)type; mi.i16_mode = (uint8_t)best_mode; mi.chroma_mode = (uint8_t)cbest; mi.cbp = (uint8_t)cbp;
        f.mbinfo[mb] = mi;
      }
    }
    }
    __syncthreads();
  }
}

int launch_intra(const FrameCtx& f, cudaStream_t st) {
  k_intra_rows<false><<<f.n_slices, 96, 0, st>>>(f);
  return 1;
}

// ---- k_scene_cut (B2V_FLAG_SCENE_CUT): once per P picture, behind its analysis (DESIGN.md §5.14; oracle/h264_scut_ref.c) ----
// One warp per macroblock: cost_intra(mb), the smallest luma SAD of Intra16x16 vertical, horizontal and DC prediction (8.3.3) formed
// from the SOURCE picture's neighbouring samples, available at the picture's edges only (no slices: an estimate, no reconstruction),
// + lambda x SCUT_INTRA_MB_BITS (no intra macroblock is free, a noise-level inter one is), and cost_inter(mb), which the analysis
// stored; while a long-term picture is a reference (B2V_FLAG_LONG_TERM_REF), the smaller of that and the cost of the long-term
// picture's zero vector, the same way (0 within the noise threshold, else SAD + 2 lambda), for every macroblock: the lean pass tries
// it only within the noise threshold, and returning content must stay P.  It runs before k_ltr_mark, so the long-term picture and
// its epoch are those this picture was analysed with.  Per block the two sums go into the picture's totals; the last block to finish
// decides: cut = SCUT_INTRA_WEIGHT x cost_intra < SCUT_INTER_WEIGHT x cost_inter.
constexpr int SCUT_WARPS = 8;
__global__ void __launch_bounds__(32 * SCUT_WARPS) k_scene_cut(FrameCtx f) {
  __shared__ unsigned long long s_intra[SCUT_WARPS], s_inter[SCUT_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int mb = blockIdx.x * SCUT_WARPS + warp;
  if (mb < f.mbw * f.mbh) {
    const int mby = mb / f.mbw, mbx = mb - mby * f.mbw, r8 = lane >> 1, c8 = (lane & 1) * 8;
    const bool top = mby > 0, left = mbx > 0;
    const uint8_t* src = f.cur + (size_t)(mby * 16 + r8) * f.cw + mbx * 16 + c8;
    const uint32_t s0 = *reinterpret_cast<const uint32_t*>(src), s1 = *reinterpret_cast<const uint32_t*>(src + 4);
    uint32_t t0 = 0, t1 = 0, l = 0;
    if (top) { const uint8_t* a = f.cur + (size_t)(mby * 16 - 1) * f.cw + mbx * 16 + c8; t0 = *reinterpret_cast<const uint32_t*>(a); t1 = *reinterpret_cast<const uint32_t*>(a + 4); }
    if (left) l = src[-c8 - 1];
    const int st = __reduce_add_sync(FULL, lane < 2 ? (int)(__vsadu4(t0, 0u) + __vsadu4(t1, 0u)) : 0);   // row 0's lanes hold the row above
    const int sl = __reduce_add_sync(FULL, (lane & 1) == 0 ? (int)l : 0);                               // one lane per row: the left column
    const uint32_t pd = rep4(top && left ? (st + sl + 16) >> 5 : top ? (st + 8) >> 4 : left ? (sl + 8) >> 4 : 128), ph = rep4((int)l);
    int best = (int)__reduce_add_sync(FULL, __vsadu4(s0, pd) + __vsadu4(s1, pd));
    if (top) best = min(best, (int)__reduce_add_sync(FULL, __vsadu4(s0, t0) + __vsadu4(s1, t1)));
    if (left) best = min(best, (int)__reduce_add_sync(FULL, __vsadu4(s0, ph) + __vsadu4(s1, ph)));
    const int lambda = me_lambda[frame_qp(f)];
    int inter = f.scut_cost[mb];
    if (f.ltr && f.ltr->epoch == f.ltr_epoch) {     // the long-term picture is a reference: its zero vector is every macroblock's candidate
      const uint8_t* lt = f.lt + (src - f.cur);
      const int s = (int)__reduce_add_sync(FULL, __vsadu4(s0, *reinterpret_cast<const uint32_t*>(lt)) + __vsadu4(s1, *reinterpret_cast<const uint32_t*>(lt + 4)));
      inter = min(inter, s <= ME_EARLY_SAD_PER_LAMBDA * lambda ? 0 : s + 2 * lambda);
    }
    if (lane == 0) { s_intra[warp] = (unsigned long long)(best + lambda * SCUT_INTRA_MB_BITS); s_inter[warp] = (unsigned long long)inter; }
  } else if (lane == 0) { s_intra[warp] = 0; s_inter[warp] = 0; }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long a = 0, b = 0;
    for (int w = 0; w < SCUT_WARPS; w++) { a += s_intra[w]; b += s_inter[w]; }
    atomicAdd(&f.scut->intra, a); atomicAdd(&f.scut->inter, b);
    __threadfence();
    if (atomicAdd(&f.scut->done, 1u) == gridDim.x - 1) {
      __threadfence();
      const unsigned long long intra = atomicExch(&f.scut->intra, 0ull), inter = atomicExch(&f.scut->inter, 0ull);
      f.scut->cut[f.pic & 1] = SCUT_INTRA_WEIGHT * intra < SCUT_INTER_WEIGHT * inter;
      f.scut->done = 0;
    }
  }
}

// k_scene_cut, then k_intra_rows on the IDR grid, which codes the picture when it was cut: two launches per P picture
int launch_scene_cut(const FrameCtx& f, cudaStream_t st) {
  k_scene_cut<<<(f.mbw * f.mbh + SCUT_WARPS - 1) / SCUT_WARPS, 32 * SCUT_WARPS, 0, st>>>(f);
  FrameCtx g = f;
  g.slice_rows = 1; g.slice_cols = f.cut_slice_cols; g.n_slices = f.cut_n_slices;
  g.slice_words = f.cut_slice_words; g.chunks_per_slice = f.cut_chunks;
  k_intra_rows<true><<<g.n_slices, 96, 0, st>>>(g);
  return 2;
}

}  // namespace b2v
