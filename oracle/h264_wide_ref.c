/*
 * h264_wide_ref.c — CPU restatement of wide-range motion (B2V_FLAG_WIDE_MOTION, include/b2video.h; DESIGN.md 5.3) on top of the
 * single-layer oracle of h264_ref.c and the droppable layers of h264_layers_ref.c, both unchanged.  TEST INFRASTRUCTURE ONLY.
 *
 * h264_layers_ref.c (and through it h264_ref.c) is compiled into this translation unit once more, its public names renamed below,
 * so that this file reaches the encoder's state and static helpers; the handle it works on is one that b2v_ref_enc_create made
 * (same source, same layout).  What this file restates for the GPU's k_coarse and the WIDE variants of k_inter_lean / k_inter_search
 * (selkies_b200/csrc/h264_inter.cu):
 *   - the decimated luma of every picture (1/4 x 1/4, each sample the rounded mean of a 4x4 block of the coded luma), kept with the
 *     reconstruction buffer the picture was coded into: keyed by that buffer's address, so the layers' buffer swaps carry it along;
 *   - one coarse vector per anchor group whose anchor's co-located SAD exceeds the early-termination threshold;
 *   - windows centred on far candidates, the anchors' second search around the coarse vector, the vector range and the wider
 *     I_PCM header budget: encode_inter_mb_wide, which is h264_ref.c encode_inter_mb with those rules;
 *   - wide_encode: h264_ref.c b2v_ref_enc_encode with the decimation and the coarse search in front of the analysis and
 *     encode_inter_mb_wide for P macroblocks; wide_layers_encode: h264_layers_ref.c b2v_ref_layers_encode around wide_encode.
 */
#define lyr_enc_create_ wide_lyr_enc_create_
#define lyr_enc_destroy_ wide_lyr_enc_destroy_
#define lyr_enc_coded_w_ wide_lyr_enc_coded_w_
#define lyr_enc_coded_h_ wide_lyr_enc_coded_h_
#define lyr_enc_recon_ wide_lyr_enc_recon_
#define lyr_enc_last_qp_ wide_lyr_enc_last_qp_
#define lyr_enc_rc_state_ wide_lyr_enc_rc_state_
#define lyr_enc_set_paintover_ wide_lyr_enc_set_paintover_
#define lyr_enc_set_idr_slice_mbs_ wide_lyr_enc_set_idr_slice_mbs_
#define lyr_enc_set_paintover_burst_ wide_lyr_enc_set_paintover_burst_
#define lyr_enc_set_stripes_ wide_lyr_enc_set_stripes_
#define lyr_enc_stripe_table_ wide_lyr_enc_stripe_table_
#define lyr_enc_max_au_ wide_lyr_enc_max_au_
#define lyr_enc_encode_ wide_lyr_enc_encode_
#define b2v_ref_layers_create wide_lyr_layers_create_
#define b2v_ref_layers_destroy wide_lyr_layers_destroy_
#define b2v_ref_layers_encode wide_lyr_layers_encode_
#include "h264_layers_ref.c"

typedef struct {
  enc_t* e;                /* the single-layer encoder (b2v_ref_enc_create) */
  layers_t* l;             /* droppable pictures: the layers (NULL without them) */
  uint8_t* dec[3];         /* decimated luma planes ... */
  const uint8_t* dec_key[3];   /* ... and the reconstruction buffer each belongs to */
  int32_t* coarse;         /* [mbs] at each anchor: its group's coarse vector (dx & 0xffff | dy << 16) or COARSE_NONE */
} wide_t;

/* ---- wide-range motion (B2V_FLAG_WIDE_MOTION; DESIGN.md 5.3; selkies_b200/csrc/h264_inter.cu k_coarse) ----
 * Vector range: a full-sample vector is usable when each component lies in [-255, 255], so that with a quarter-sample refinement
 * (+-3/4) every coded component lies in [-1024, 1023] quarter samples: the range the SPS asserts (VUI log2_max_mv_length_horizontal
 * = log2_max_mv_length_vertical = 10), inside Table A-1's MaxVmvR of every level the SPS writes (3.1 and up: [-512, 511.75]) and
 * the horizontal [-2048, 2047.75]. */
#define MV_MAX_FULL 255
static int mv_ok(int kx, int ky) { return kx >= -MV_MAX_FULL && kx <= MV_MAX_FULL && ky >= -MV_MAX_FULL && ky <= MV_MAX_FULL; }
/* coarse search of an anchor group, decimated samples: dx in [-32, 31], dy in [-64, 63] (x4: +-128 and +-256 luma samples).  The
 * +-16 search around the scaled vector skips the candidates outside MV_MAX_FULL. */
#define WM_DX 32
#define WM_DY 64
#define COARSE_NONE 0x7fffffff
#define WM_MVD_BITS 48     /* header budget of a P macroblock in a wide-motion picture: 48 more bits for two mvd of up to +-2046 */

static uint8_t* dec_plane(wide_t* w, const uint8_t* buf, int create) {
  for (int i = 0; i < 3; i++) if (w->dec_key[i] == buf) return w->dec[i];
  if (!create) return NULL;
  for (int i = 0; i < 3; i++) if (!w->dec_key[i]) { w->dec_key[i] = buf; return w->dec[i]; }
  abort();                 /* more than three reconstruction buffers */
}
/* the decimated luma: each sample the rounded mean of a 4x4 block of the coded luma */
static void decimate(const enc_t* e, const uint8_t* y, uint8_t* d) {
  const int dw = e->cw / 4, dh = e->ch / 4;
  for (int j = 0; j < dh; j++)
    for (int i = 0; i < dw; i++) {
      int s = 0;
      for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) s += y[(size_t)(4 * j + r) * e->cw + 4 * i + c];
      d[(size_t)j * dw + i] = (uint8_t)((s + 8) >> 4);
    }
}
/* one coarse vector per anchor group whose anchor's co-located SAD exceeds the early-termination threshold: the group's decimated
 * block (4x4 decimated samples per macroblock of the group) against the reference picture's decimated plane, at every position
 * inside the picture and the band, minimum of (SAD, |dx| + |dy|, dy, dx) */
static void coarse_search(wide_t* w, const uint8_t* cur_nv12, int qp) {
  enc_t* e = w->e;
  const uint8_t* dc = dec_plane(w, e->recon[e->cur], 0); const uint8_t* dr = dec_plane(w, e->recon[e->cur ^ 1], 0);
  const uint8_t* refy = plane_y(e, e->cur ^ 1);
  const int dw = e->cw / 4, lambda = me_lambda[qp];
  for (int i = 0; i < e->mbw * e->mbh; i++) w->coarse[i] = COARSE_NONE;
#pragma omp parallel for schedule(dynamic, 1)
  for (int mby = 0; mby < e->mbh; mby++)
    for (int mbx = 0; mbx < e->mbw; mbx++) {
      if (!is_anchor(e, mbx, mby) || !dr) continue;
      int sad0 = 0;
      for (int r = 0; r < 16; r++)
        for (int c = 0; c < 16; c++) sad0 += iabs(cur_nv12[(size_t)(mby * 16 + r) * e->cw + mbx * 16 + c] - refy[(size_t)(mby * 16 + r) * e->cw + mbx * 16 + c]);
      if (sad0 <= ME_EARLY_SAD_PER_LAMBDA * lambda) continue;
      int br0, br1; band_rows(e, mby, &br0, &br1);
      const int gx0 = mbx / 4 * 4, gy0 = br0 + (mby - br0) / 4 * 4;
      const int gx1 = gx0 + 4 < e->mbw ? gx0 + 4 : e->mbw, gy1 = gy0 + 4 < br1 ? gy0 + 4 : br1;
      const int X0 = 4 * gx0, Y0 = 4 * gy0, W = 4 * (gx1 - gx0), H = 4 * (gy1 - gy0);
      uint64_t best = ~0ull;
      for (int dy = -WM_DY; dy < WM_DY; dy++)
        for (int dx = -WM_DX; dx < WM_DX; dx++) {
          if (X0 + dx < 0 || X0 + dx + W > dw || Y0 + dy < 4 * br0 || Y0 + dy + H > 4 * br1) continue;
          int sad = 0;
          for (int r = 0; r < H; r++)
            for (int c = 0; c < W; c++) sad += iabs(dc[(size_t)(Y0 + r) * dw + X0 + c] - dr[(size_t)(Y0 + dy + r) * dw + X0 + dx + c]);
          const uint64_t key = (uint64_t)sad << 20 | (uint64_t)(iabs(dx) + iabs(dy)) << 13 | (uint64_t)(dy + 64) << 6 | (uint64_t)(dx + 32);
          if (key < best) best = key;
        }
      if (best != ~0ull) w->coarse[mby * e->mbw + mbx] = (int32_t)(((int)(best & 63) - 32) & 0xffff) | (int32_t)(((int)((best >> 6) & 127) - 64) * 65536);
    }
}
/* the 48x48 window centred on the full-sample vector (wx,wy): win[j][i] = ref(x0-16+wx+i, y0-16+wy+j), clamped (8.4.2.2.1) */
static void stage_win(const enc_t* e, const uint8_t* refy, int x0, int y0, int wx, int wy, int ylo, int yhi, uint8_t win[48][48]) {
  const int xs = x0 - 16 + wx;
  for (int j = 0; j < 48; j++) {
    const uint8_t* rr = refy + (size_t)clip3(ylo, yhi, y0 - 16 + wy + j) * e->cw;
    if (xs >= 0 && xs + 48 <= e->cw) memcpy(win[j], rr + xs, 48);
    else for (int i = 0; i < 48; i++) win[j][i] = rr[clip3(0, e->cw - 1, xs + i)];
  }
}



static int in_colocated_window(int cdx, int cdy) { return cdx >= -15 && cdx <= 14 && cdy >= -15 && cdy <= 15; }
/* (cdx,cdy) relative to a window centred on the full-sample vector (wx,wy): costs are those of the real vector (wx+cdx, wy+cdy),
 * the key's index is relative to the window.  Every window but a wide-motion one is centred on (0,0). */
static int try_candidate_at(const uint8_t cy[256], uint8_t win[48][48], int cdx, int cdy, int wx, int wy, int lambda, int sad0, uint32_t* key) {
  if (!in_colocated_window(cdx, cdy)) return 0;
  uint32_t kc = 0, kmin = 0xffffffffu;
  for (int j = -1; j <= 1; j++)
    for (int i = -1; i <= 1; i++) {
      int sad = 0;
      for (int r = 0; r < 16; r++) for (int c = 0; c < 16; c++) sad += iabs(cy[r * 16 + c] - win[16 + cdy + j + r][16 + cdx + i + c]);
      const uint32_t cost = (uint32_t)(sad + lambda * (se_bits(4 * (wx + cdx + i)) + se_bits(4 * (wy + cdy + j))));
      const uint32_t k = (cost << 11) | (uint32_t)((cdy + j + 16) * 32 + (cdx + i + 16));
      if (i == 0 && j == 0) kc = k; else if (k < kmin) kmin = k;
    }
  const int sadc = (int)(kc >> 11) - lambda * (se_bits(4 * (wx + cdx)) + se_bits(4 * (wy + cdy)));
  const uint32_t key0 = ((uint32_t)(sad0 + 2 * lambda) << 11) | (16 * 32 + 16);     /* the zero vector's own key */
  if (sadc <= ME_PRED_SAD_FACTOR * ME_EARLY_SAD_PER_LAMBDA * lambda && kc < kmin && kc <= key0) { *key = kc; return 1; }
  return 0;
}


/* make_pcm_if_too_big with the header budget of a wide-motion picture: WM_MVD_BITS more for the mvd */
static void make_pcm_if_too_big_wide(enc_t* e, mb_t* m, const uint8_t* cur_nv12, int mbx, int mby) {
  if (mb_bits_estimate(m) + WM_MVD_BITS <= MB_BITS_LIMIT) return;
  uint8_t* ry = plane_y(e, e->cur); uint8_t* ruv = plane_uv(e, e->cur);
  const uint8_t* cuv = cur_nv12 + (size_t)e->cw * e->ch;
  for (int r = 0; r < 16; r++) memcpy(ry + (size_t)(mby * 16 + r) * e->cw + mbx * 16, cur_nv12 + (size_t)(mby * 16 + r) * e->cw + mbx * 16, 16);
  for (int r = 0; r < 8; r++) memcpy(ruv + (size_t)(mby * 8 + r) * e->cw + mbx * 16, cuv + (size_t)(mby * 8 + r) * e->cw + mbx * 16, 16);
  m->type = 2; m->cbp = 0; m->mv[0] = m->mv[1] = 0;
  memset(m->nnz_l, 16, sizeof m->nnz_l); memset(m->nnz_c, 16, sizeof m->nnz_c);
}

/* h264_ref.c encode_inter_mb with wide-range motion */
static void encode_inter_mb_wide(wide_t* w, const uint8_t* cur_nv12, int mbx, int mby, int qp) {
  enc_t* e = w->e;
  mb_t* m = &e->mbs[mby * e->mbw + mbx];
  const int prev_type = m->type, prev_mvx = m->mv[0], prev_mvy = m->mv[1];   /* this macroblock in the previous picture */
  memset(m, 0, sizeof *m);
  m->type = 1;
  uint8_t cy[256], cc[2][64];
  load_cur(cur_nv12, e->cw, e->ch, mbx, mby, cy, cc);
  const uint8_t* refy = plane_y(e, e->cur ^ 1); const uint8_t* refuv = plane_uv(e, e->cur ^ 1);
  int x0 = mbx * 16, y0 = mby * 16, lambda = me_lambda[qp];
  int br0, br1; band_rows(e, mby, &br0, &br1);
  const int ylo = br0 * 16, yhi = br1 * 16 - 1;      /* a band's decoder pads at the band's own edges */
  uint32_t best = 0xffffffffu; int bdx = 0, bdy = 0;
  /* reference samples the search can touch, with picture-edge clamping (8.4.2.2.1): win[j][i] = ref(x0-16+i, y0-16+j) */
  uint8_t win[48][48];
  for (int j = 0; j < 48; j++) {
    const uint8_t* rr = refy + (size_t)clip3(ylo, yhi, y0 - 16 + j) * e->cw;
    if (x0 >= 16 && x0 + 32 <= e->cw) memcpy(win[j], rr + x0 - 16, 48);
    else for (int i = 0; i < 48; i++) win[j][i] = rr[clip3(0, e->cw - 1, x0 - 16 + i)];
  }
  /* zero-motion early termination: when the co-located block already matches to within the quantisation noise
   * expected at this QP (SAD <= 96*lambda), the search is skipped and mv = (0,0) */
  int sad0 = 0;
  for (int r = 0; r < 16; r++) for (int c = 0; c < 16; c++) sad0 += iabs(cy[r * 16 + c] - win[16 + r][16 + c]);
  int search = sad0 > ME_EARLY_SAD_PER_LAMBDA * lambda;
  /* temporal-predictor early termination: the vector this macroblock had in the previous picture, rounded to full samples
   * (scrolling and panning content repeats it).  Accepted without the exhaustive search when its SAD is within 4x the noise
   * threshold AND it is a strict local minimum of the cost over its 8 full-sample neighbours (all inside the search range)
   * AND it costs less than the zero vector (otherwise a stale vector could survive on a scene that has become static);
   * quarter-sample refinement then runs as after a search. */
  int pred_hit = 0, src_mvx = 0, src_mvy = 0, dyr = 16, tried_zero = 0;      /* src_mv: the vector the accepted candidate was derived from */
  /* the centre of the window `win` holds (full samples); bdx, bdy are relative to it.  Only wide-range motion moves it: a candidate
   * outside the co-located window's test range is tested in a window centred on (its x rounded down to a multiple of 4, its y) */
  int wx = 0, wy = 0;
  if (search && prev_type == 1) {
    const int cdx = asr(prev_mvx + 2, 2), cdy = asr(prev_mvy + 2, 2);
    tried_zero = !(cdx | cdy);
    if (!in_colocated_window(cdx, cdy) && mv_ok(cdx, cdy)) {
      wx = cdx & ~3; wy = cdy; stage_win(e, refy, x0, y0, wx, wy, ylo, yhi, win);
      if (try_candidate_at(cy, win, cdx - wx, cdy - wy, wx, wy, lambda, sad0, &best)) { search = 0; pred_hit = 1; bdx = cdx - wx; bdy = cdy - wy; src_mvx = prev_mvx; src_mvy = prev_mvy; }
    } else if ((!tried_zero || !e->no_zcand) && try_candidate_at(cy, win, cdx, cdy, 0, 0, lambda, sad0, &best)) { search = 0; pred_hit = 1; bdx = cdx; bdy = cdy; src_mvx = prev_mvx; src_mvy = prev_mvy; }
  }
  /* anchor predictor: the vector the anchor of this macroblock's 4x4 group found in THIS picture (anchors run first) */
  if (search && !e->no_anchor && !is_anchor(e, mbx, mby)) {
    int ax, ay; anchor_of(e, mbx, mby, &ax, &ay);
    const mb_t* a = &e->mbs[ay * e->mbw + ax];
    const int cdx = asr(a->me_mv[0] + 2, 2), cdy = asr(a->me_mv[1] + 2, 2);
    const int skip_zero = !(cdx | cdy) && (tried_zero || e->no_zcand);      /* the zero vector is not tested twice */
    const int shifted = !in_colocated_window(cdx, cdy) && mv_ok(cdx, cdy);
    if (shifted) { wx = cdx & ~3; wy = cdy; stage_win(e, refy, x0, y0, wx, wy, ylo, yhi, win); }
    else if (wx | wy) { wx = wy = 0; stage_win(e, refy, x0, y0, 0, 0, ylo, yhi, win); }
    if (!skip_zero && try_candidate_at(cy, win, cdx - wx, cdy - wy, wx, wy, lambda, sad0, &best)) { search = 0; pred_hit = 1; bdx = cdx - wx; bdy = cdy - wy; src_mvx = a->me_mv[0]; src_mvy = a->me_mv[1]; }
    /* new content: the anchor's exhaustive search found no match worth the name and this macroblock's co-located block is as far
     * off — another 1089-candidate search would only pick the least bad of the noise.  The search shrinks to the five rows
     * around dy = 0 (160 candidates: most of what picking a minimum among noise buys, for a sixth of the work). */
    else if (a->me_bad && sad0 >= ME_REFINE_MAX_SAD && !e->no_newcontent) dyr = ME_NEWCONTENT_DY;
  }
  if (search && (wx | wy)) { wx = wy = 0; stage_win(e, refy, x0, y0, 0, 0, ylo, yhi, win); }
  for (int dy = -dyr; search && dy <= dyr; dy++)
    for (int dx = -16; dx <= 15; dx++) {
      int sad = 0;
      for (int r = 0; r < 16; r++) {
        const uint8_t* rr = &win[dy + 16 + r][dx + 16];
        for (int c = 0; c < 16; c++) sad += iabs(cy[r * 16 + c] - rr[c]);
      }
      uint32_t cost = (uint32_t)(sad + lambda * (se_bits(4 * dx) + se_bits(4 * dy)));
      uint32_t key = (cost << 11) | (uint32_t)((dy + 16) * 32 + (dx + 16));
      if (key < best) { best = key; bdx = dx; bdy = dy; }
    }
  /* wide-range motion, an anchor that searched: the same search in the window centred on its group's coarse vector x 4, unless the
   * co-located search covered that vector with the 4 samples either way that one decimated sample spans (|x| <= 12, |y| <= 12 and
   * x <= 11).  The cheaper result by true cost wins; on equal cost the co-located window. */
  if (search && is_anchor(e, mbx, mby) && w->coarse[mby * e->mbw + mbx] != COARSE_NONE) {
    const int32_t cv = w->coarse[mby * e->mbw + mbx];
    const int cx = 4 * (int)(int16_t)(cv & 0xffff), cyv = 4 * (cv >> 16);
    if (cx < -12 || cx > 11 || cyv < -12 || cyv > 12) {
      uint8_t win2[48][48];
      stage_win(e, refy, x0, y0, cx, cyv, ylo, yhi, win2);
      uint32_t best2 = 0xffffffffu; int b2x = 0, b2y = 0;
      for (int dy = -16; dy <= 16; dy++)
        for (int dx = -16; dx <= 15; dx++) {
          if (!mv_ok(cx + dx, cyv + dy)) continue;
          int sad = 0;
          for (int r = 0; r < 16; r++) for (int c = 0; c < 16; c++) sad += iabs(cy[r * 16 + c] - win2[dy + 16 + r][dx + 16 + c]);
          const uint32_t key = ((uint32_t)(sad + lambda * (se_bits(4 * (cx + dx)) + se_bits(4 * (cyv + dy)))) << 11) | (uint32_t)((dy + 16) * 32 + (dx + 16));
          if (key < best2) { best2 = key; b2x = dx; b2y = dy; }
        }
      if ((best2 >> 11) < (best >> 11)) { best = best2; bdx = b2x; bdy = b2y; wx = cx; wy = cyv; memcpy(win, win2, sizeof win); }
    }
  }
  /* ---- quarter-sample refinement (8.4.2.2.1).  Around the best full-sample position (only when its 6-tap support
   * [-3,+18] lies inside the 48x48 window, i.e. |dx|,|dy| <= 13, and the search ran): the half-sample planes
   *   b1 = E - 5F + 20G + 20H - 5I + J (unrounded), b = clip((b1+16)>>5), h likewise vertically, j = clip((6-tap of b1 + 512)>>10)
   * are built once; stage H tries the 8 half-sample neighbours, stage Q the 8 quarter-sample neighbours of the stage-H
   * winner; cost = SAD + lambda*(bits(mvx)+bits(mvy) + 4 if fractional), key = cost<<4 | candidate index (0 = centre wins ties). */
  int mvx = 4 * (wx + bdx), mvy = 4 * (wy + bdy);
  uint8_t py[256], pc[2][64];
  int have_planes = 0;
  static const int8_t nb8[8][2] = { {-1,-1}, {0,-1}, {1,-1}, {-1,0}, {1,0}, {-1,1}, {0,1}, {1,1} };
  uint8_t Gp[22][22], bq[18][17], hq[17][18], jq[17][17];   /* Gp[v+3][u+3], bq[v+1][u+1], hq[v+1][u+1], jq[v+1][u+1] */
  /* not worth refining when the full-sample match is already within the quantisation noise of this QP */
  const int sad_int = (int)(best >> 11) - lambda * (se_bits(4 * (wx + bdx)) + se_bits(4 * (wy + bdy)));
  m->me_bad = (search || pred_hit) && sad_int >= ME_REFINE_MAX_SAD;     /* however the vector was found: nothing here matches */
  /* a predictor hit whose previous vector was full-sample is not refined again: the previous refinement already preferred it */
  const int pred_frac = pred_hit && ((src_mvx | src_mvy) & 3);
  /* ... nor when it is hopeless (mean absolute difference of 32 per sample and more: new content, nothing to polish) */
  if ((search || pred_frac) && iabs(bdx) <= 13 && iabs(bdy) <= 13 && sad_int > ME_EARLY_SAD_PER_LAMBDA * lambda && sad_int < ME_REFINE_MAX_SAD) {
    int16_t b1[22][17];
    const int ox = 16 + bdx, oy = 16 + bdy;
    for (int v = -3; v <= 18; v++) for (int u = -3; u <= 18; u++) Gp[v + 3][u + 3] = win[oy + v][ox + u];
#define GW(u, v) ((int)Gp[(v) + 3][(u) + 3])
    for (int v = -3; v <= 18; v++)
      for (int u = -1; u <= 15; u++) b1[v + 3][u + 1] = (int16_t)(GW(u - 2, v) - 5 * GW(u - 1, v) + 20 * GW(u, v) + 20 * GW(u + 1, v) - 5 * GW(u + 2, v) + GW(u + 3, v));
    for (int v = -1; v <= 16; v++) for (int u = -1; u <= 15; u++) bq[v + 1][u + 1] = (uint8_t)clip1((b1[v + 3][u + 1] + 16) >> 5);
    for (int v = -1; v <= 15; v++)
      for (int u = -1; u <= 16; u++)
        hq[v + 1][u + 1] = (uint8_t)clip1((GW(u, v - 2) - 5 * GW(u, v - 1) + 20 * GW(u, v) + 20 * GW(u, v + 1) - 5 * GW(u, v + 2) + GW(u, v + 3) + 16) >> 5);
    for (int v = -1; v <= 15; v++)
      for (int u = -1; u <= 15; u++)
        jq[v + 1][u + 1] = (uint8_t)clip1((b1[v + 1][u + 1] - 5 * b1[v + 2][u + 1] + 20 * b1[v + 3][u + 1] + 20 * b1[v + 4][u + 1] - 5 * b1[v + 5][u + 1] + b1[v + 6][u + 1] + 512) >> 10);
    have_planes = 1;
    int cx = 0, cyq = 0;                      /* offset from the full-sample position, quarter units */
    for (int stage = 0; stage < 2; stage++) {
      const int step = stage == 0 ? 2 : 1;
      uint32_t bestk = 0xffffffffu; int bi = 0;
      for (int i = 0; i <= 8; i++) {
        const int qx = cx + (i ? nb8[i - 1][0] * step : 0), qy = cyq + (i ? nb8[i - 1][1] * step : 0);
        uint8_t pr[256];
        luma_mc_planes(Gp, bq, hq, jq, qx, qy, pr);
        const uint32_t cost = (uint32_t)(sad_n(cy, pr, 256) + lambda * (se_bits(4 * (wx + bdx) + qx) + se_bits(4 * (wy + bdy) + qy) + (((qx | qy) & 3) ? ME_FRAC_PENALTY_BITS : 0)));
        const uint32_t key = (cost << 4) | (uint32_t)i;
        if (key < bestk) { bestk = key; bi = i; }
      }
      if (bi) { cx += nb8[bi - 1][0] * step; cyq += nb8[bi - 1][1] * step; }
    }
    mvx += cx; mvy += cyq;
    luma_mc_planes(Gp, bq, hq, jq, cx, cyq, py);
#undef GW
  }
  m->mv[0] = m->me_mv[0] = (int16_t)mvx; m->mv[1] = m->me_mv[1] = (int16_t)mvy;
  /* prediction: luma from the planes above, or a full-sample copy; chroma bilinear 1/8 (8.4.2.2.2) */
  if (!have_planes)
    for (int r = 0; r < 16; r++)
      for (int c = 0; c < 16; c++) py[r * 16 + c] = refy[(size_t)clip3(ylo, yhi, y0 + wy + bdy + r) * e->cw + clip3(0, e->cw - 1, x0 + wx + bdx + c)];
  int mvcx = mvx, mvcy = mvy, xi = asr(mvcx, 3), yi = asr(mvcy, 3), xf = mvcx & 7, yf = mvcy & 7;
  int cwc = e->cw / 2;
  for (int r = 0; r < 8; r++)
    for (int c = 0; c < 8; c++) {
      int xa = clip3(0, cwc - 1, mbx * 8 + xi + c), xb = clip3(0, cwc - 1, mbx * 8 + xi + c + 1);
      int ya = clip3(ylo / 2, yhi / 2, mby * 8 + yi + r), yb = clip3(ylo / 2, yhi / 2, mby * 8 + yi + r + 1);
      for (int k = 0; k < 2; k++) {
        int A = refuv[(size_t)ya * e->cw + xa * 2 + k], B = refuv[(size_t)ya * e->cw + xb * 2 + k];
        int C = refuv[(size_t)yb * e->cw + xa * 2 + k], D = refuv[(size_t)yb * e->cw + xb * 2 + k];
        pc[k][r * 8 + c] = (uint8_t)(((8 - xf) * (8 - yf) * A + xf * (8 - yf) * B + (8 - xf) * yf * C + xf * yf * D + 32) >> 6);
      }
    }
  uint8_t* ry = plane_y(e, e->cur);
  int cbp = 0;
  /* coefficient decimation (encoder-side, as x264's dct-decimate): a block's score is 9 if any |level| > 1, else the sum
   * over its +-1 levels of {3,2,2,1,1,1,0...}[zeros just below it in scan order]; an 8x8 quadrant whose four scores sum
   * to < 4 is zeroed, and the whole luma when the macroblock total is < 6 — a few isolated +-1 cost more bits than they repair */
  int score[16], s8[4] = {0, 0, 0, 0}, smb = 0;
  for (int b = 0; b < 16; b++) {
    int bx = blk_x[b] * 4, by = blk_y[b] * 4, res[16], dummy;
    for (int i = 0; i < 16; i++) { int p = (by + (i >> 2)) * 16 + bx + (i & 3); res[i] = cy[p] - py[p]; }
    tq4x4(res, qp, 0, 0, m->coef[1 + b], &dummy);
    int sc = 0, zeros = 0, big = 0;
    for (int k = 0; k < 16; k++) {
      int v = m->coef[1 + b][k];
      if (!v) { zeros++; continue; }
      if (iabs(v) > 1) big = 1;
      sc += zeros == 0 ? 3 : zeros <= 2 ? 2 : zeros <= 5 ? 1 : 0;
      zeros = 0;
    }
    score[b] = big ? 9 : sc;
    s8[b >> 2] += score[b]; smb += score[b];
  }
  for (int b = 0; b < 16; b++) {
    int bx = blk_x[b] * 4, by = blk_y[b] * 4;
    if (s8[b >> 2] < 4 || smb < 6) memset(m->coef[1 + b], 0, sizeof m->coef[1 + b]);
    int n = count_nz(m->coef[1 + b], 0, 16);
    m->nnz_l[blk_y[b] * 4 + blk_x[b]] = (uint8_t)n;
    if (n) cbp |= 1 << (b >> 2);
    int resid[16];
    recon4x4(m->coef[1 + b], qp, 0, 0, resid);
    for (int i = 0; i < 16; i++) {
      int y = by + (i >> 2), x = bx + (i & 3);
      ry[(size_t)(y0 + y) * e->cw + x0 + x] = (uint8_t)clip1(py[y * 16 + x] + resid[i]);
    }
  }
  int cbp_c = code_chroma(e, m, mbx, mby, qp, 0, cc, pc);
  m->cbp = (uint8_t)(cbp | (cbp_c << 4));
  make_pcm_if_too_big_wide(e, m, cur_nv12, mbx, mby);
}


/* h264_ref.c b2v_ref_enc_encode with the decimation and the coarse search in front of the analysis, encode_inter_mb_wide for P macroblocks */
static int64_t wide_encode(wide_t* w, const uint8_t* cur_nv12, int idr, int rc_mode, int qp_fixed, int64_t target_bits, uint8_t* out) {
  enc_t* e = w->e;
  int mbs = e->mbw * e->mbh;
  const int k = (int)(e->pic & 1);
  const struct rcfb used = e->fb[k];                         /* the controller state after picture pic-2 */
  const int qp = rc_frame_qp(e, &used, idr, rc_mode, qp_fixed, target_bits);
  e->cur ^= 1;
  e->pic_rows = idr ? 1 : e->slice_rows; e->pic_cols = idr ? e->seg_cols : e->mbw;
  const int nsl = pic_n_slices(e);
  if (idr) { e->frame_num = 0; }
  /* this picture's decimated luma, then the anchors' coarse vectors against the reference's */
  decimate(e, cur_nv12, dec_plane(w, e->recon[e->cur], 1));
  if (!idr) coarse_search(w, cur_nv12, qp);
  else for (int i = 0; i < mbs; i++) w->coarse[i] = COARSE_NONE;      /* nothing reads it in an IDR; b2v_ref_wide_coarse reports none */
  /* phase A: analysis + reconstruction.  Intra: macroblocks of a slice are sequential (left/top
   * dependencies), slices are independent.  Inter: every macroblock is independent. */
  if (idr) {
#pragma omp parallel for schedule(dynamic, 1)
    for (int s = 0; s < nsl; s++) {
      const rect_t r = slice_rect(e, s);
      for (int mby = r.row0; mby < r.row1; mby++)
        for (int mbx = r.x0; mbx < r.x1; mbx++) encode_intra_mb(e, cur_nv12, mbx, mby, qp);
    }
  } else {
    /* anchors first (their vectors are candidates for the rest of their groups), then everybody else */
    for (int pass = 0; pass < 2; pass++) {
#pragma omp parallel for schedule(dynamic, 1)
      for (int mby = 0; mby < e->mbh; mby++)
        for (int mbx = 0; mbx < e->mbw; mbx++) if (is_anchor(e, mbx, mby) == (pass == 0)) encode_inter_mb_wide(w, cur_nv12, mbx, mby, qp);
    }
  }
  /* phase B: entropy coding per slice, then concatenation */
  uint8_t* skip = (uint8_t*)calloc(mbs, 1);
  const rect_t full = slice_rect(e, 0);        /* slice 0 is a full-size slice */
  const size_t per = (size_t)(full.row1 - full.row0) * (full.x1 - full.x0) * 1024 + 256;
  uint8_t* tmp = (uint8_t*)malloc(per * nsl);
  size_t* lens = (size_t*)calloc(nsl, sizeof(size_t));
  int64_t* sbits = (int64_t*)calloc(nsl, sizeof(int64_t));
#pragma omp parallel for schedule(dynamic, 1)
  for (int s = 0; s < nsl; s++) lens[s] = code_slice(e, s, idr, qp, skip, tmp + per * s, &sbits[s]);
  size_t o = 0; int64_t bits = 0;
  if (!e->stripe_rows) {
    if (idr) { memcpy(out + o, e->sps, e->sps_len); o += e->sps_len; memcpy(out + o, e->pps, e->pps_len); o += e->pps_len; }
    for (int s = 0; s < nsl; s++) { memcpy(out + o, tmp + per * s, lens[s]); o += lens[s]; bits += sbits[s]; }
  } else {
    /* bands back to back, each a complete access unit of its own stream; a P band whose macroblocks were all skipped
     * is flagged not-coded (the caller drops it) and its frame_num does not advance */
    for (int t = 0; t < e->n_stripes; t++) {
      const int r0 = t * e->stripe_rows, r1 = r0 + e->stripe_rows > e->mbh ? e->mbh : r0 + e->stripe_rows;
      const int last = t == e->n_stripes - 1;
      const size_t o0 = o;
      if (idr) { memcpy(out + o, e->sps_band[last], e->sps_band_len[last]); o += e->sps_band_len[last]; memcpy(out + o, e->pps, e->pps_len); o += e->pps_len; }
      for (int s = 0; s < nsl; s++) {
        const int row0 = slice_rect(e, s).row0;
        if (row0 >= r0 && row0 < r1) { memcpy(out + o, tmp + per * s, lens[s]); o += lens[s]; bits += sbits[s]; }
      }
      int coded = idr;
      for (int i = r0 * e->mbw; i < r1 * e->mbw && !coded; i++) coded |= !skip[i];
      e->stripe_tab[t][0] = (int32_t)o0; e->stripe_tab[t][1] = (int32_t)(o - o0); e->stripe_tab[t][2] = coded;
      e->stripe_fn[t] = idr ? 1 : (e->stripe_fn[t] + (coded ? 1 : 0)) & 255;
    }
  }
  uint8_t* skip_copy = skip;
  free(tmp); free(lens); free(sbits);
  { int coded = 0; for (int i = 0; i < mbs; i++) coded |= !skip_copy[i]; free(skip_copy);
    struct rcfb init; memset(&init, 0, sizeof init); init.qp = -1;
    const struct rcfb prev = e->pic > 0 ? e->fb[k ^ 1] : init;
    /* RBSP bits of the slices: known before the byte stream is assembled */
    /* + 40 bits per slice NAL (start code, NAL header): what the wire carries beyond the RBSP, to a good approximation */
    rc_step(e, &e->fb[k], &prev, &used, bits + 40LL * nsl, qp, idr, coded, rc_mode, target_bits); }
  e->last_qp = qp; e->last_bits = (int64_t)o * 8; e->pic++;
  if (idr) e->idr_count++;
  e->frame_num = (e->frame_num + 1) & 255;
  return (int64_t)o;
}

/* h264_layers_ref.c b2v_ref_layers_encode with wide_encode in place of the single-layer encode: droppable and wide-range motion */
static int64_t wide_layers_encode(wide_t* w, const uint8_t* cur_nv12, int idr, int rc_mode, int qp_fixed, int64_t target_bits, uint8_t* out) {
  layers_t* l = w->l;
  enc_t* e = l->e;
  if (idr) { l->since_idr = 0; l->frame_num = 0; }
  const int is_ref = idr || (l->since_idr & 1) == 0;
  const int ref_dist = l->last_was_ref ? 1 : 2;
  /* reference: the last reference picture, in `spare` while the last picture is a non-reference one */
  if (!l->last_was_ref) { uint8_t* t = e->recon[e->cur]; e->recon[e->cur] = l->spare; l->spare = t; }
  if (!idr && ref_dist != l->last_ref_dist) {
    const int mbs = e->mbw * e->mbh;
    for (int i = 0; i < mbs; i++)
      if (e->mbs[i].type == 1) {
        e->mbs[i].mv[0] = (int16_t)scale_mv(e->mbs[i].mv[0], ref_dist, l->last_ref_dist);
        e->mbs[i].mv[1] = (int16_t)scale_mv(e->mbs[i].mv[1], ref_dist, l->last_ref_dist);
      }
  }
  const int k = (int)(e->pic & 1);
  struct rcfb init; memset(&init, 0, sizeof init); init.qp = -1;
  const struct rcfb used = e->fb[k], prev = e->pic > 0 ? e->fb[k ^ 1] : init;
  e->frame_num = l->frame_num;
  int64_t n = wide_encode(w, cur_nv12, idr, rc_mode, qp_fixed, target_bits, out);
  if (!is_ref) {
    /* the slices again as slices of a non-reference picture, then the rate-control step again on their bits */
    const int nsl = pic_n_slices(e), mbs = e->mbw * e->mbh;
    uint8_t* skip = (uint8_t*)calloc(mbs, 1);
    const size_t per = (size_t)e->pic_rows * e->mbw * 1024 + 256;
    uint8_t* tmp = (uint8_t*)malloc(per * nsl);
    size_t* lens = (size_t*)calloc(nsl, sizeof(size_t));
    int64_t* sbits = (int64_t*)calloc(nsl, sizeof(int64_t));
#pragma omp parallel for schedule(dynamic, 1)
    for (int s = 0; s < nsl; s++) lens[s] = code_slice_nonref(e, s, e->last_qp, l->frame_num, skip, tmp + per * s, &sbits[s]);
    size_t o = 0; int64_t bits = 0;
    for (int s = 0; s < nsl; s++) { memcpy(out + o, tmp + per * s, lens[s]); o += lens[s]; bits += sbits[s]; }
    int coded = 0;
    for (int i = 0; i < mbs; i++) coded |= !skip[i];
    free(skip); free(tmp); free(lens); free(sbits);
    rc_step(e, &e->fb[k], &prev, &used, bits + 40LL * nsl, e->last_qp, 0, coded, rc_mode, target_bits);
    e->last_bits = (int64_t)o * 8;
    n = (int64_t)o;
    /* keep the reference (the buffer this picture predicted from) for the next picture */
    uint8_t* t = e->recon[e->cur ^ 1]; e->recon[e->cur ^ 1] = l->spare; l->spare = t;
  } else {
    l->frame_num = (l->frame_num + 1) & 255;
  }
  l->last_was_ref = is_ref; l->last_ref_dist = ref_dist;
  l->since_idr++;
  return n;
}


/* wide-range motion on the encoder `h` (b2v_ref_enc_create), before its first picture; droppable: with two temporal layers
 * (h264_layers_ref.c rules; NULL in striped mode, as there).  Encode through b2v_ref_wide_encode from then on. */
void* b2v_ref_wide_create(void* h, int droppable) {
  enc_t* e = (enc_t*)h;
  wide_t* w = (wide_t*)calloc(1, sizeof *w);
  w->e = e;
  if (droppable && !(w->l = (layers_t*)wide_lyr_layers_create_(h))) { free(w); return NULL; }
  for (int i = 0; i < 3; i++) w->dec[i] = (uint8_t*)calloc((size_t)(e->cw / 4) * (e->ch / 4), 1);
  w->coarse = (int32_t*)calloc((size_t)e->mbw * e->mbh, sizeof(int32_t));
  return w;
}
void b2v_ref_wide_destroy(void* wh) {
  wide_t* w = (wide_t*)wh;
  if (!w) return;
  wide_lyr_layers_destroy_(w->l);
  for (int i = 0; i < 3; i++) free(w->dec[i]);
  free(w->coarse); free(w);
}
/* b2v_ref_enc_encode (or b2v_ref_layers_encode) with wide-range motion; returns the access unit's size */
int64_t b2v_ref_wide_encode(void* wh, const uint8_t* cur_nv12, int idr, int rc_mode, int qp_fixed, int64_t target_bits, uint8_t* out) {
  wide_t* w = (wide_t*)wh;
  return w->l ? wide_layers_encode(w, cur_nv12, idr, rc_mode, qp_fixed, target_bits, out) : wide_encode(w, cur_nv12, idr, rc_mode, qp_fixed, target_bits, out);
}
/* the last picture's coarse table (mbw x mbh int32: at an anchor its group's dx & 0xffff | dy << 16, else COARSE_NONE) */
void b2v_ref_wide_coarse(void* wh, int32_t* out) {
  const wide_t* w = (const wide_t*)wh;
  memcpy(out, w->coarse, sizeof(int32_t) * w->e->mbw * w->e->mbh);
}
/* the last picture's decimated luma ((cw / 4) x (ch / 4)), the plane kept with the reconstruction buffer it was coded into */
void b2v_ref_wide_decimated(void* wh, uint8_t* out) {
  wide_t* w = (wide_t*)wh;
  memcpy(out, dec_plane(w, w->e->recon[w->e->cur], 0), (size_t)(w->e->cw / 4) * (w->e->ch / 4));
}
