/*
 * h264_ltr_ref.c — CPU restatement of the long-term reference picture (B2V_FLAG_LONG_TERM_REF, include/b2video.h; DESIGN.md 5.13)
 * on top of the oracles of h264_ref.c and h264_wide_ref.c, both unchanged.  TEST INFRASTRUCTURE ONLY.
 *
 * h264_wide_ref.c (and through it h264_layers_ref.c and h264_ref.c) is compiled into this translation unit once more, every public
 * name renamed below, so that this file reaches the encoder's state and static helpers; the handle it works on is one that
 * b2v_ref_enc_create made (same source, same layout).  What this file restates for the GPU's k_ltr_mark, the LTR variants of
 * k_inter_lean and the entropy stage (selkies_b200/csrc/h264_inter.cu, h264_entropy.cu):
 *   - the SPS with max_num_ref_frames 2 and max_dec_frame_buffering 2;
 *   - the long-term buffer, outside the two reconstruction buffers;
 *   - changed(k) and the marking rule, and the copy of picture k-1's reconstruction into the buffer when picture k marks;
 *   - the zero-vector long-term test, placed where the lean pass makes it: after the zero-vector exit and the lean pass's
 *     temporal-predictor exit fail (a hit on a full-sample predictor of a macroblock whose window lies inside the picture);
 *     such a macroblock is coded by the unchanged macroblock coder with the long-term picture as its reference, where it takes the
 *     zero-vector exit, and gets refIdx 1 (mb_t.i16_mode, unused in P macroblocks);
 *   - refIdx-aware motion-vector prediction (8.4.1.3) and P_Skip (8.4.1.1, refIdx 0 only), ref_idx_l0, the slice-header override
 *     and the memory-management operations: ltr_code_slice, h264_ref.c code_slice with those rules;
 *   - the rate-control step on those slices' bits: ltr_encode, h264_wide_ref.c wide_encode with the rules above, wide-range
 *     motion on or off.
 * Full frame only: striped encoders are refused, and there are no droppable pictures.
 */
#define wide_lyr_enc_create_ ltr_lyr_enc_create_
#define wide_lyr_enc_destroy_ ltr_lyr_enc_destroy_
#define wide_lyr_enc_coded_w_ ltr_lyr_enc_coded_w_
#define wide_lyr_enc_coded_h_ ltr_lyr_enc_coded_h_
#define wide_lyr_enc_recon_ ltr_lyr_enc_recon_
#define wide_lyr_enc_last_qp_ ltr_lyr_enc_last_qp_
#define wide_lyr_enc_rc_state_ ltr_lyr_enc_rc_state_
#define wide_lyr_enc_set_paintover_ ltr_lyr_enc_set_paintover_
#define wide_lyr_enc_set_idr_slice_mbs_ ltr_lyr_enc_set_idr_slice_mbs_
#define wide_lyr_enc_set_paintover_burst_ ltr_lyr_enc_set_paintover_burst_
#define wide_lyr_enc_set_stripes_ ltr_lyr_enc_set_stripes_
#define wide_lyr_enc_stripe_table_ ltr_lyr_enc_stripe_table_
#define wide_lyr_enc_max_au_ ltr_lyr_enc_max_au_
#define wide_lyr_enc_encode_ ltr_lyr_enc_encode_
#define wide_lyr_layers_create_ ltr_lyr_layers_create_
#define wide_lyr_layers_destroy_ ltr_lyr_layers_destroy_
#define wide_lyr_layers_encode_ ltr_lyr_layers_encode_
#define b2v_ref_wide_create ltr_wide_create_
#define b2v_ref_wide_destroy ltr_wide_destroy_
#define b2v_ref_wide_encode ltr_wide_encode_
#define b2v_ref_wide_coarse ltr_wide_coarse_
#define b2v_ref_wide_decimated ltr_wide_decimated_
#include "h264_wide_ref.c"

/* the marking rule: picture k marks picture k-1 long-term when changed(k) >= max(ceil(mbs / LTR_CHANGED_MIN_DIV),
 * LTR_CHANGED_RATIO * changed(k-1)) (h264_inter.cu k_ltr_mark) */
#define LTR_CHANGED_MIN_DIV 64
#define LTR_CHANGED_RATIO 8

typedef struct {
  enc_t* e;                /* the single-layer encoder (b2v_ref_enc_create) */
  wide_t* w;               /* decimated planes and coarse vectors: used with wide-range motion only */
  int wide;
  uint8_t* lt;             /* the long-term reference picture's reconstruction (NV12, coded size) */
  int lt_valid;            /* it is a reference: marked since the last IDR */
  int prev_changed;        /* changed(k-1); an IDR picture counts every macroblock */
  uint8_t* cls;            /* [mbs] lean-pass class of each macroblock of the picture being coded (LEAN_*) */
  int32_t state[4];        /* the last picture: two references, marks, MMCO 1, changed */
} ltr_t;

enum { LEAN_ZERO = 0, LEAN_PRED = 1, LEAN_LT = 2, LEAN_QUEUED = 3 };

/* 7.3.2.1 SPS of h264_ref.c build_sps with two reference frames */
static int build_sps_ltr(uint8_t* dst, int mbw, int mbh, int crop_r, int crop_b) {
  bitw_t b; bw_init(&b);
  bw_put(&b, 8, 66); bw_put(&b, 8, 0xC0); bw_put(&b, 8, level_idc_for(mbw, mbh));
  bw_ue(&b, 0); bw_ue(&b, 4); bw_ue(&b, 2);
  bw_ue(&b, 2);                 /* max_num_ref_frames: the previous picture and the long-term one */
  bw_put(&b, 1, 0);
  bw_ue(&b, mbw - 1); bw_ue(&b, mbh - 1);
  bw_put(&b, 1, 1); bw_put(&b, 1, 1);
  if (crop_r || crop_b) { bw_put(&b, 1, 1); bw_ue(&b, 0); bw_ue(&b, crop_r); bw_ue(&b, 0); bw_ue(&b, crop_b); }
  else bw_put(&b, 1, 0);
  bw_put(&b, 1, 1); bw_put(&b, 1, 0); bw_put(&b, 1, 0);
  bw_put(&b, 1, 1); bw_put(&b, 3, 5); bw_put(&b, 1, 0); bw_put(&b, 1, 1);
  bw_put(&b, 8, 1); bw_put(&b, 8, 1); bw_put(&b, 8, 1);
  bw_put(&b, 1, 1); bw_ue(&b, 1); bw_ue(&b, 1);
  bw_put(&b, 1, 0); bw_put(&b, 1, 0); bw_put(&b, 1, 0); bw_put(&b, 1, 0);
  bw_put(&b, 1, 1); bw_put(&b, 1, 1);
  bw_ue(&b, 0); bw_ue(&b, 0);
  bw_ue(&b, 10); bw_ue(&b, 10);
  bw_ue(&b, 0);
  bw_ue(&b, 2);                 /* max_dec_frame_buffering */
  bw_trailing(&b);
  int n = (int)nal_write(dst, 1, 3, 7, b.buf, b.pos);
  bw_free(&b);
  return n;
}

/* The lean pass's decision for one macroblock (h264_inter.cu k_inter_lean), before anything of this picture is coded: the zero-
 * vector exit, the temporal-predictor exit it takes (a full-sample predictor of a macroblock whose window lies inside the picture;
 * the rest is left to the search pass), then, while a long-term picture exists, the zero vector into it. */
static int lean_class(ltr_t* l, const uint8_t* cur_nv12, int mbx, int mby, int qp) {
  enc_t* e = l->e;
  const mb_t* m = &e->mbs[mby * e->mbw + mbx];
  const uint8_t* refy = plane_y(e, e->cur ^ 1);
  const int x0 = mbx * 16, y0 = mby * 16, lambda = me_lambda[qp];
  int br0, br1; band_rows(e, mby, &br0, &br1);
  const int ylo = br0 * 16, yhi = br1 * 16 - 1;
  uint8_t cy[256], cc[2][64];
  load_cur(cur_nv12, e->cw, e->ch, mbx, mby, cy, cc);
  int sad0 = 0, sad_lt = 0;
  for (int r = 0; r < 16; r++)
    for (int c = 0; c < 16; c++) {
      sad0 += iabs(cy[r * 16 + c] - refy[(size_t)(y0 + r) * e->cw + x0 + c]);
      sad_lt += iabs(cy[r * 16 + c] - l->lt[(size_t)(y0 + r) * e->cw + x0 + c]);
    }
  if (sad0 <= ME_EARLY_SAD_PER_LAMBDA * lambda) return LEAN_ZERO;
  if (m->type == 1) {
    int cdx = asr(m->mv[0] + 2, 2), cdy = asr(m->mv[1] + 2, 2), wx = 0, wy = 0;
    int in = in_colocated_window(cdx, cdy);
    if (l->wide && !in && mv_ok(cdx, cdy)) { wx = cdx & ~3; wy = cdy; in = 1; }
    const int inside = x0 - 16 + wx >= 0 && x0 + 32 + wx <= e->cw;
    if (in && inside && !((m->mv[0] | m->mv[1]) & 3)) {
      uint8_t win[48][48]; uint32_t key;
      stage_win(e, refy, x0, y0, wx, wy, ylo, yhi, win);
      if (try_candidate_at(cy, win, cdx - wx, cdy - wy, wx, wy, lambda, sad0, &key)) return LEAN_PRED;
    }
  }
  if (l->lt_valid && sad_lt <= ME_EARLY_SAD_PER_LAMBDA * lambda) return LEAN_LT;
  return LEAN_QUEUED;
}

/* 8.4.1.3 / 8.4.1.1 with refIdx: a neighbour's refIdx is mb_t.i16_mode of a P_L0_16x16 macroblock, -1 for intra or unavailable */
static void ltr_neighbours(const enc_t* e, int mbx, int mby, int av[3], int ref[3], int mv[3][2]) {
  int top = avail_top(e, mby);
  int nx[3] = { mbx - 1, mbx, mbx + 1 }, ny[3] = { mby, mby - 1, mby - 1 };
  av[0] = avail_left(e, mbx); av[1] = top; av[2] = top && mbx + 1 < e->mbw;
  if (!av[2]) { nx[2] = mbx - 1; av[2] = top && mbx > 0; }
  for (int i = 0; i < 3; i++) {
    mv[i][0] = mv[i][1] = 0; ref[i] = -1;
    if (av[i]) {
      const mb_t* n = &e->mbs[ny[i] * e->mbw + nx[i]];
      if (n->type == 1) { ref[i] = n->i16_mode; mv[i][0] = n->mv[0]; mv[i][1] = n->mv[1]; }
    }
  }
}
static void ltr_mv_pred16(const enc_t* e, int mbx, int mby, int refidx, int out[2]) {
  int av[3], ref[3], mv[3][2];
  ltr_neighbours(e, mbx, mby, av, ref, mv);
  if (!av[1] && !av[2] && av[0]) { out[0] = mv[0][0]; out[1] = mv[0][1]; return; }
  const int cnt = (ref[0] == refidx) + (ref[1] == refidx) + (ref[2] == refidx);
  if (cnt == 1) { const int i = ref[0] == refidx ? 0 : ref[1] == refidx ? 1 : 2; out[0] = mv[i][0]; out[1] = mv[i][1]; return; }
  out[0] = median3(mv[0][0], mv[1][0], mv[2][0]);
  out[1] = median3(mv[0][1], mv[1][1], mv[2][1]);
}
static void ltr_mv_pred_skip(const enc_t* e, int mbx, int mby, int out[2]) {
  out[0] = out[1] = 0;
  if (!avail_left(e, mbx) || !avail_top(e, mby)) return;
  const mb_t* a = &e->mbs[mby * e->mbw + mbx - 1]; const mb_t* b = &e->mbs[(mby - 1) * e->mbw + mbx];
  if ((a->type == 1 && a->i16_mode == 0 && a->mv[0] == 0 && a->mv[1] == 0) || (b->type == 1 && b->i16_mode == 0 && b->mv[0] == 0 && b->mv[1] == 0)) return;
  ltr_mv_pred16(e, mbx, mby, 0, out);
}

/* 7.3.3 slice header: h264_ref.c write_slice_header with the override (two active references) and the marking operations */
static void ltr_slice_header(const enc_t* e, bitw_t* b, int first_mb, int idr, int qp, int frame_num, int active, int mark, int drop_st) {
  bw_ue(b, first_mb);
  bw_ue(b, idr ? 7 : 5);
  bw_ue(b, 0);
  bw_put(b, 8, frame_num & 255);
  if (idr) bw_ue(b, e->idr_count & 15);
  if (!idr) {
    if (active) { bw_put(b, 1, 1); bw_ue(b, 1); }   /* num_ref_idx_active_override_flag, num_ref_idx_l0_active_minus1 */
    else bw_put(b, 1, 0);
    bw_put(b, 1, 0);                             /* ref_pic_list_modification_flag_l0 */
  }
  if (idr) { bw_put(b, 1, 0); bw_put(b, 1, 0); }    /* no_output_of_prior_pics_flag, long_term_reference_flag */
  else if (mark) {
    bw_put(b, 1, 1);                             /* adaptive_ref_pic_marking_mode_flag */
    if (drop_st) { bw_ue(b, 1); bw_ue(b, 1); }   /* MMCO 1: the short-term picture two back (picNumX = CurrPicNum - 2) */
    bw_ue(b, 4); bw_ue(b, 1);                    /* MMCO 4: max_long_term_frame_idx_plus1 = 1 */
    bw_ue(b, 3); bw_ue(b, 0); bw_ue(b, 0);       /* MMCO 3: the previous picture to long_term_frame_idx 0 */
    bw_ue(b, 0);                                 /* MMCO 0 */
  } else bw_put(b, 1, 0);
  bw_se(b, qp - 26);
  bw_ue(b, 1);
}

/* h264_ref.c code_slice (full frame) with ltr_slice_header, ref_idx_l0 and refIdx-aware prediction */
static size_t ltr_code_slice(enc_t* e, int s, int idr, int qp, int active, int mark, int drop_st, uint8_t* skip, uint8_t* out, int64_t* bits) {
  bitw_t b; bw_init(&b);
  const rect_t r = slice_rect(e, s);
  ltr_slice_header(e, &b, r.row0 * e->mbw + r.x0, idr, qp, idr ? 0 : e->frame_num, active, mark, drop_st);
  int skip_run = 0;
  for (int mby = r.row0; mby < r.row1; mby++)
    for (int mbx = r.x0; mbx < r.x1; mbx++) {
      const mb_t* m = &e->mbs[mby * e->mbw + mbx];
      if (!idr) {
        int sp[2];
        ltr_mv_pred_skip(e, mbx, mby, sp);
        if (m->type == 1 && m->i16_mode == 0 && m->cbp == 0 && m->mv[0] == sp[0] && m->mv[1] == sp[1]) { skip[mby * e->mbw + mbx] = 1; skip_run++; continue; }
        bw_ue(&b, skip_run); skip_run = 0;
      }
      if (m->type == 2) {
        bw_ue(&b, idr ? 25 : 30);
        if (b.nacc) bw_put(&b, 8 - b.nacc, 0);
        const uint8_t* ry = plane_y(e, e->cur); const uint8_t* ruv = plane_uv(e, e->cur);
        for (int y = 0; y < 16; y++) for (int x = 0; x < 16; x++) bw_put(&b, 8, ry[(size_t)(mby * 16 + y) * e->cw + mbx * 16 + x]);
        for (int k = 0; k < 2; k++)
          for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) bw_put(&b, 8, ruv[(size_t)(mby * 8 + y) * e->cw + (mbx * 8 + x) * 2 + k]);
        continue;
      }
      if (m->type == 3) {
        bw_ue(&b, idr ? 0 : 5);
        for (int blk = 0; blk < 16; blk++) {
          int bx = blk_x[blk], by = blk_y[blk], mode = m->i4_modes[by * 4 + bx], pm = i4_pred_mode(e, mbx, mby, bx, by);
          if (mode == pm) bw_put(&b, 1, 1);
          else { bw_put(&b, 1, 0); bw_put(&b, 3, mode < pm ? mode : mode - 1); }
        }
        bw_ue(&b, m->chroma_mode);
        bw_ue(&b, cbp_to_codenum_intra[m->cbp]);
        if (m->cbp) bw_se(&b, 0);
        write_residual(e, &b, skip, m, mbx, mby);
        continue;
      }
      if (m->type == 0) {
        int t = 1 + m->i16_mode + 4 * (m->cbp >> 4) + ((m->cbp & 15) ? 12 : 0);
        bw_ue(&b, idr ? t : t + 5);
        bw_ue(&b, m->chroma_mode);
        bw_se(&b, 0);
      } else {
        int mvp[2];
        ltr_mv_pred16(e, mbx, mby, m->i16_mode, mvp);
        bw_ue(&b, 0);                          /* P_L0_16x16 */
        if (active) bw_put(&b, 1, m->i16_mode ? 0 : 1);   /* ref_idx_l0: te(v), range 1 */
        bw_se(&b, m->mv[0] - mvp[0]); bw_se(&b, m->mv[1] - mvp[1]);
        bw_ue(&b, cbp_to_codenum_inter[m->cbp]);
        if (m->cbp) bw_se(&b, 0);
      }
      write_residual(e, &b, skip, m, mbx, mby);
    }
  if (skip_run) bw_ue(&b, skip_run);
  *bits = (int64_t)bw_bits(&b);
  bw_trailing(&b);
  size_t n = nal_write(out, r.row0 == 0 && r.x0 == 0 && !idr, idr ? 3 : 2, idr ? 5 : 1, b.buf, b.pos);
  bw_free(&b);
  return n;
}

static void ltr_inter_mb(ltr_t* l, const uint8_t* cur_nv12, int mbx, int mby, int qp) {
  if (l->wide) encode_inter_mb_wide(l->w, cur_nv12, mbx, mby, qp); else encode_inter_mb(l->e, cur_nv12, mbx, mby, qp);
}

/* h264_wide_ref.c wide_encode (full frame) with the long-term reference */
static int64_t ltr_encode(ltr_t* l, const uint8_t* cur_nv12, int idr, int rc_mode, int qp_fixed, int64_t target_bits, uint8_t* out) {
  enc_t* e = l->e;
  const int mbs = e->mbw * e->mbh;
  const int k = (int)(e->pic & 1);
  const struct rcfb used = e->fb[k];
  const int qp = rc_frame_qp(e, &used, idr, rc_mode, qp_fixed, target_bits);
  e->cur ^= 1;
  e->pic_rows = idr ? 1 : e->slice_rows; e->pic_cols = idr ? e->seg_cols : e->mbw;
  const int nsl = pic_n_slices(e);
  if (idr) { e->frame_num = 0; }
  if (l->wide) {
    decimate(e, cur_nv12, dec_plane(l->w, e->recon[e->cur], 1));
    if (!idr) coarse_search(l->w, cur_nv12, qp);
  }
  const int active = !idr && l->lt_valid;
  int changed = mbs, mark = 0;
  if (idr) {
#pragma omp parallel for schedule(dynamic, 1)
    for (int s = 0; s < nsl; s++) {
      const rect_t r = slice_rect(e, s);
      for (int mby = r.row0; mby < r.row1; mby++)
        for (int mbx = r.x0; mbx < r.x1; mbx++) encode_intra_mb(e, cur_nv12, mbx, mby, qp);
    }
  } else {
    /* the lean pass's decisions, from the previous picture's records, before any of them is overwritten */
    changed = 0;
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : changed)
    for (int mby = 0; mby < e->mbh; mby++)
      for (int mbx = 0; mbx < e->mbw; mbx++) {
        const int c = lean_class(l, cur_nv12, mbx, mby, qp);
        l->cls[mby * e->mbw + mbx] = (uint8_t)c;
        changed += c != LEAN_ZERO;
      }
    /* the long-term macroblocks: the macroblock coder with the long-term picture as its reference takes the zero-vector exit */
    uint8_t* st = e->recon[e->cur ^ 1];
    e->recon[e->cur ^ 1] = l->lt;
#pragma omp parallel for schedule(dynamic, 1)
    for (int mby = 0; mby < e->mbh; mby++)
      for (int mbx = 0; mbx < e->mbw; mbx++)
        if (l->cls[mby * e->mbw + mbx] == LEAN_LT) {
          ltr_inter_mb(l, cur_nv12, mbx, mby, qp);
          mb_t* m = &e->mbs[mby * e->mbw + mbx];
          if (m->type == 1) m->i16_mode = 1;
        }
    e->recon[e->cur ^ 1] = st;
    /* anchors first (their vectors are candidates for the rest of their groups), then everybody else */
    for (int pass = 0; pass < 2; pass++) {
#pragma omp parallel for schedule(dynamic, 1)
      for (int mby = 0; mby < e->mbh; mby++)
        for (int mbx = 0; mbx < e->mbw; mbx++)
          if (l->cls[mby * e->mbw + mbx] != LEAN_LT && is_anchor(e, mbx, mby) == (pass == 0)) ltr_inter_mb(l, cur_nv12, mbx, mby, qp);
    }
    const int lo = (mbs + LTR_CHANGED_MIN_DIV - 1) / LTR_CHANGED_MIN_DIV, hi = LTR_CHANGED_RATIO * l->prev_changed;
    mark = changed >= (lo > hi ? lo : hi);
  }
  const int drop_st = mark && !active;
  uint8_t* skip = (uint8_t*)calloc(mbs, 1);
  const rect_t full = slice_rect(e, 0);
  const size_t per = (size_t)(full.row1 - full.row0) * (full.x1 - full.x0) * 1024 + 256;
  uint8_t* tmp = (uint8_t*)malloc(per * nsl);
  size_t* lens = (size_t*)calloc(nsl, sizeof(size_t));
  int64_t* sbits = (int64_t*)calloc(nsl, sizeof(int64_t));
#pragma omp parallel for schedule(dynamic, 1)
  for (int s = 0; s < nsl; s++) lens[s] = ltr_code_slice(e, s, idr, qp, active, mark, drop_st, skip, tmp + per * s, &sbits[s]);
  size_t o = 0; int64_t bits = 0;
  if (idr) { memcpy(out + o, e->sps, e->sps_len); o += e->sps_len; memcpy(out + o, e->pps, e->pps_len); o += e->pps_len; }
  for (int s = 0; s < nsl; s++) { memcpy(out + o, tmp + per * s, lens[s]); o += lens[s]; bits += sbits[s]; }
  free(tmp); free(lens); free(sbits);
  { int coded = 0; for (int i = 0; i < mbs; i++) coded |= !skip[i]; free(skip);
    struct rcfb init; memset(&init, 0, sizeof init); init.qp = -1;
    const struct rcfb prev = e->pic > 0 ? e->fb[k ^ 1] : init;
    rc_step(e, &e->fb[k], &prev, &used, bits + 40LL * nsl, qp, idr, coded, rc_mode, target_bits); }
  /* marking takes effect after this picture: picture k-1's reconstruction, intact until the next picture is coded into its buffer */
  if (mark) { memcpy(l->lt, e->recon[e->cur ^ 1], (size_t)e->cw * e->ch * 3 / 2); l->lt_valid = 1; }
  if (idr) l->lt_valid = 0;
  l->prev_changed = changed;
  l->state[0] = active; l->state[1] = mark; l->state[2] = drop_st; l->state[3] = changed;
  e->last_qp = qp; e->last_bits = (int64_t)o * 8; e->pic++;
  if (idr) e->idr_count++;
  e->frame_num = (e->frame_num + 1) & 255;
  return (int64_t)o;
}

/* the long-term reference on the encoder `h` (b2v_ref_enc_create, full frame), before its first picture: its SPS is rewritten with
 * two reference frames.  wide: with wide-range motion (h264_wide_ref.c rules).  NULL in striped mode.  Encode through
 * b2v_ref_ltr_encode from then on. */
void* b2v_ref_ltr_create(void* h, int wide) {
  enc_t* e = (enc_t*)h;
  if (e->stripe_rows) return NULL;
  ltr_t* l = (ltr_t*)calloc(1, sizeof *l);
  l->e = e; l->wide = wide;
  l->w = (wide_t*)ltr_wide_create_(h, 0);
  l->lt = (uint8_t*)calloc((size_t)e->cw * e->ch * 3 / 2, 1);
  l->cls = (uint8_t*)calloc((size_t)e->mbw * e->mbh, 1);
  l->prev_changed = e->mbw * e->mbh;
  e->sps_len = build_sps_ltr(e->sps, e->mbw, e->mbh, (e->cw - e->width) / 2, (e->ch - e->height) / 2);
  return l;
}
void b2v_ref_ltr_destroy(void* lh) {
  ltr_t* l = (ltr_t*)lh;
  if (!l) return;
  ltr_wide_destroy_(l->w);
  free(l->lt); free(l->cls); free(l);
}
int64_t b2v_ref_ltr_encode(void* lh, const uint8_t* cur_nv12, int idr, int rc_mode, int qp_fixed, int64_t target_bits, uint8_t* out) {
  return ltr_encode((ltr_t*)lh, cur_nv12, idr, rc_mode, qp_fixed, target_bits, out);
}
/* the last picture: {two active references, marks the previous picture, MMCO 1, changed}; the long-term picture (NULL while none) */
void b2v_ref_ltr_state(void* lh, int32_t* out) { memcpy(out, ((ltr_t*)lh)->state, sizeof ((ltr_t*)lh)->state); }
const uint8_t* b2v_ref_ltr_picture(void* lh) { ltr_t* l = (ltr_t*)lh; return l->lt_valid ? l->lt : NULL; }
