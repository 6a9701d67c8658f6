/*
 * h264_scut_ref.c — CPU restatement of scene cuts (B2V_FLAG_SCENE_CUT, include/b2video.h; DESIGN.md 5.14) on top of the oracles of
 * h264_ref.c, h264_layers_ref.c, h264_wide_ref.c and h264_ltr_ref.c, all unchanged.  TEST INFRASTRUCTURE ONLY.
 *
 * h264_ltr_ref.c (and through it the other three) is compiled into this translation unit once more, every public name renamed below,
 * so that this file reaches the encoders' state and static helpers; the handles it works on are ones that b2v_ref_enc_create and
 * b2v_ref_ltr_create made (same sources, same layouts).  scut_encode is h264_ltr_ref.c ltr_encode with:
 *   - the droppable layers of h264_layers_ref.c (reference selection, predictor scaling, the frame_num rule, nal_ref_idc 0 and no
 *     dec_ref_pic_marking() in a non-reference picture), so that every permitted combination of the opt-in flags has a model;
 *   - the long-term reference optional: without it no long-term picture is ever marked and the SPS stays the single-reference one;
 *   - the decision (selkies_b200/csrc/h264_intra.cu k_scene_cut) after the P analysis: cost_inter, the sum over macroblocks of the
 *     luma SAD of the chosen prediction (motion compensation 8.4.2.2.1 at the vector motion estimation chose, or the long-term
 *     picture at the zero vector) + lambda x (se(v) bits of both components + ME_FRAC_PENALTY_BITS for a fractional vector), 0 for a
 *     macroblock whose SAD is within the zero-motion exit's threshold, and while a long-term picture is a reference the smaller of that
 *     and the same cost of the long-term picture's zero vector, against cost_intra, the sum over macroblocks of the smallest
 *     luma SAD of Intra16x16 vertical, horizontal and DC prediction from the source picture's neighbours (available inside the
 *     picture) + lambda x SCUT_INTRA_MB_BITS; cut when SCUT_INTRA_WEIGHT x cost_intra < SCUT_INTER_WEIGHT x cost_inter;
 *   - a cut picture: every macroblock coded again by the IDR coder (encode_intra_mb) in the IDR slice grid, at the P picture's QP, over
 *     the P analysis's records and reconstruction; its slices are I slices of a non-IDR picture (scut_code_slice) with the P
 *     picture's frame_num, nal_ref_idc and marking.
 * Full frame only: striped encoders are refused.
 */
#define ltr_lyr_enc_create_ scut_lyr_enc_create_
#define ltr_lyr_enc_destroy_ scut_lyr_enc_destroy_
#define ltr_lyr_enc_coded_w_ scut_lyr_enc_coded_w_
#define ltr_lyr_enc_coded_h_ scut_lyr_enc_coded_h_
#define ltr_lyr_enc_recon_ scut_lyr_enc_recon_
#define ltr_lyr_enc_last_qp_ scut_lyr_enc_last_qp_
#define ltr_lyr_enc_rc_state_ scut_lyr_enc_rc_state_
#define ltr_lyr_enc_set_paintover_ scut_lyr_enc_set_paintover_
#define ltr_lyr_enc_set_idr_slice_mbs_ scut_lyr_enc_set_idr_slice_mbs_
#define ltr_lyr_enc_set_paintover_burst_ scut_lyr_enc_set_paintover_burst_
#define ltr_lyr_enc_set_stripes_ scut_lyr_enc_set_stripes_
#define ltr_lyr_enc_stripe_table_ scut_lyr_enc_stripe_table_
#define ltr_lyr_enc_max_au_ scut_lyr_enc_max_au_
#define ltr_lyr_enc_encode_ scut_lyr_enc_encode_
#define ltr_lyr_layers_create_ scut_lyr_layers_create_
#define ltr_lyr_layers_destroy_ scut_lyr_layers_destroy_
#define ltr_lyr_layers_encode_ scut_lyr_layers_encode_
#define ltr_wide_create_ scut_wide_create_
#define ltr_wide_destroy_ scut_wide_destroy_
#define ltr_wide_encode_ scut_wide_encode_
#define ltr_wide_coarse_ scut_wide_coarse_
#define ltr_wide_decimated_ scut_wide_decimated_
#define b2v_ref_ltr_create scut_ltr_create_
#define b2v_ref_ltr_destroy scut_ltr_destroy_
#define b2v_ref_ltr_encode scut_ltr_encode_
#define b2v_ref_ltr_state scut_ltr_state_
#define b2v_ref_ltr_picture scut_ltr_picture_
#include "h264_ltr_ref.c"

/* the rule (selkies_b200/csrc/h264_common.cuh) */
#define SCUT_INTRA_WEIGHT 1
#define SCUT_INTER_WEIGHT 1
#define SCUT_INTRA_MB_BITS 16

typedef struct {
  ltr_t* l;                /* the long-term layer: its long-term state with LONG_TERM_REF, its lean classes and wide planes always */
  int own_l, ltr_on;
  layers_t* y;             /* droppable pictures: the layers (NULL without them) */
  int64_t state[4];        /* the last picture: cut, cost_intra, cost_inter (0 for an IDR picture), lambda of its QP */
} scut_t;

/* 8.4.2.2.1 luma sample interpolation of the whole picture `ref` (cw x ch, samples outside clamped to the picture) */
static int ref_at(const uint8_t* ref, int cw, int ch, int x, int y) { return ref[(size_t)clip3(0, ch - 1, y) * cw + clip3(0, cw - 1, x)]; }
static int tap6(int e, int f, int g, int h, int i, int j) { return e - 5 * f + 20 * g + 20 * h - 5 * i + j; }
static int b1_at(const uint8_t* r, int cw, int ch, int x, int y) {
  return tap6(ref_at(r, cw, ch, x - 2, y), ref_at(r, cw, ch, x - 1, y), ref_at(r, cw, ch, x, y), ref_at(r, cw, ch, x + 1, y), ref_at(r, cw, ch, x + 2, y), ref_at(r, cw, ch, x + 3, y));
}
static int h1_at(const uint8_t* r, int cw, int ch, int x, int y) {
  return tap6(ref_at(r, cw, ch, x, y - 2), ref_at(r, cw, ch, x, y - 1), ref_at(r, cw, ch, x, y), ref_at(r, cw, ch, x, y + 1), ref_at(r, cw, ch, x, y + 2), ref_at(r, cw, ch, x, y + 3));
}
static int half_b(const uint8_t* r, int cw, int ch, int x, int y) { return clip1((b1_at(r, cw, ch, x, y) + 16) >> 5); }
static int half_h(const uint8_t* r, int cw, int ch, int x, int y) { return clip1((h1_at(r, cw, ch, x, y) + 16) >> 5); }
static int half_j(const uint8_t* r, int cw, int ch, int x, int y) {
  return clip1((tap6(b1_at(r, cw, ch, x, y - 2), b1_at(r, cw, ch, x, y - 1), b1_at(r, cw, ch, x, y), b1_at(r, cw, ch, x, y + 1), b1_at(r, cw, ch, x, y + 2), b1_at(r, cw, ch, x, y + 3)) + 512) >> 10);
}
/* the predicted luma sample at full-sample position (x, y) and fractional offset (xf, yf) (Table 8-12) */
static int luma_sample(const uint8_t* r, int cw, int ch, int x, int y, int xf, int yf) {
#define AVG(a, b) (((a) + (b) + 1) >> 1)
  const int G = ref_at(r, cw, ch, x, y);
  switch (yf * 4 + xf) {
    case 0: return G;
    case 1: return AVG(G, half_b(r, cw, ch, x, y));
    case 2: return half_b(r, cw, ch, x, y);
    case 3: return AVG(half_b(r, cw, ch, x, y), ref_at(r, cw, ch, x + 1, y));
    case 4: return AVG(G, half_h(r, cw, ch, x, y));
    case 5: return AVG(half_b(r, cw, ch, x, y), half_h(r, cw, ch, x, y));
    case 6: return AVG(half_b(r, cw, ch, x, y), half_j(r, cw, ch, x, y));
    case 7: return AVG(half_b(r, cw, ch, x, y), half_h(r, cw, ch, x + 1, y));
    case 8: return half_h(r, cw, ch, x, y);
    case 9: return AVG(half_h(r, cw, ch, x, y), half_j(r, cw, ch, x, y));
    case 10: return half_j(r, cw, ch, x, y);
    case 11: return AVG(half_j(r, cw, ch, x, y), half_h(r, cw, ch, x + 1, y));
    case 12: return AVG(ref_at(r, cw, ch, x, y + 1), half_h(r, cw, ch, x, y));
    case 13: return AVG(half_h(r, cw, ch, x, y), half_b(r, cw, ch, x, y + 1));
    case 14: return AVG(half_j(r, cw, ch, x, y), half_b(r, cw, ch, x, y + 1));
    default: return AVG(half_h(r, cw, ch, x + 1, y), half_b(r, cw, ch, x, y + 1));
  }
#undef AVG
}

/* cost_inter of one analysed macroblock: its prediction's luma SAD + lambda x the bits of its vector, 0 within the zero-motion exit's
 * threshold; while a long-term picture is a reference (active), the smaller of that and the same cost of its zero vector */
static int64_t inter_cost(const scut_t* s, const uint8_t* cur_nv12, int mbx, int mby, int qp, int active) {
  const ltr_t* l = s->l; const enc_t* e = l->e;
  const mb_t* m = &e->mbs[mby * e->mbw + mbx];
  const int lt = l->cls[mby * e->mbw + mbx] == LEAN_LT;
  const int mvx = lt ? 0 : m->me_mv[0], mvy = lt ? 0 : m->me_mv[1];
  const uint8_t* ref = lt ? l->lt : e->recon[e->cur ^ 1];
  int64_t sad = 0;
  for (int r = 0; r < 16; r++)
    for (int c = 0; c < 16; c++) {
      const int x = mbx * 16 + c, y = mby * 16 + r;
      sad += iabs(cur_nv12[(size_t)y * e->cw + x] - luma_sample(ref, e->cw, e->ch, x + (mvx >> 2), y + (mvy >> 2), mvx & 3, mvy & 3));
    }
  const int64_t thr = ME_EARLY_SAD_PER_LAMBDA * me_lambda[qp];
  int64_t cost = sad <= thr ? 0 : sad + (int64_t)me_lambda[qp] * (se_bits(mvx) + se_bits(mvy) + (((mvx | mvy) & 3) ? ME_FRAC_PENALTY_BITS : 0));
  if (active) {      /* the long-term picture's zero vector, a candidate of every macroblock while it is a reference */
    int64_t sl = 0;
    for (int r = 0; r < 16; r++)
      for (int c = 0; c < 16; c++) sl += iabs(cur_nv12[(size_t)(mby * 16 + r) * e->cw + mbx * 16 + c] - l->lt[(size_t)(mby * 16 + r) * e->cw + mbx * 16 + c]);
    const int64_t c_lt = sl <= thr ? 0 : sl + 2 * (int64_t)me_lambda[qp];
    if (c_lt < cost) cost = c_lt;
  }
  return cost;
}

/* cost_intra of one macroblock: min over Intra16x16 vertical, horizontal, DC (8.3.3) of the luma SAD, from the source's neighbours,
 * + lambda x SCUT_INTRA_MB_BITS */
static int64_t intra_cost(const enc_t* e, const uint8_t* cur_nv12, int mbx, int mby, int qp) {
  const uint8_t* y = cur_nv12;
  const int x0 = mbx * 16, y0 = mby * 16, top = mby > 0, left = mbx > 0;
  int st = 0, sl = 0;
  for (int i = 0; i < 16; i++) {
    if (top) st += y[(size_t)(y0 - 1) * e->cw + x0 + i];
    if (left) sl += y[(size_t)(y0 + i) * e->cw + x0 - 1];
  }
  const int dc = top && left ? (st + sl + 16) >> 5 : top ? (st + 8) >> 4 : left ? (sl + 8) >> 4 : 128;
  int sv = 0, sh = 0, sd = 0;
  for (int r = 0; r < 16; r++)
    for (int c = 0; c < 16; c++) {
      const int v = y[(size_t)(y0 + r) * e->cw + x0 + c];
      if (top) sv += iabs(v - y[(size_t)(y0 - 1) * e->cw + x0 + c]);
      if (left) sh += iabs(v - y[(size_t)(y0 + r) * e->cw + x0 - 1]);
      sd += iabs(v - dc);
    }
  int best = sd;
  if (top && sv < best) best = sv;
  if (left && sh < best) best = sh;
  return best + (int64_t)me_lambda[qp] * SCUT_INTRA_MB_BITS;
}

/* 7.3.3 slice header and 7.3.4 slice data of slice s of the picture just analysed: ltr_code_slice with I slices of a non-IDR picture
 * (intra: slice_type 7, no override, no mb_skip_run, the I-slice mb_type table) and with non-reference pictures (ref = 0: nal_ref_idc 0,
 * no dec_ref_pic_marking()) */
static size_t scut_code_slice(enc_t* e, int s, int idr, int intra, int ref, int qp, int active, int mark, int drop_st, uint8_t* skip, uint8_t* out, int64_t* bits) {
  bitw_t b; bw_init(&b);
  const rect_t r = slice_rect(e, s);
  bw_ue(&b, r.row0 * e->mbw + r.x0);
  bw_ue(&b, intra ? 7 : 5);
  bw_ue(&b, 0);
  bw_put(&b, 8, (idr ? 0 : e->frame_num) & 255);
  if (idr) bw_ue(&b, e->idr_count & 15);
  if (!intra) {
    if (active) { bw_put(&b, 1, 1); bw_ue(&b, 1); } else bw_put(&b, 1, 0);
    bw_put(&b, 1, 0);
  }
  if (idr) { bw_put(&b, 1, 0); bw_put(&b, 1, 0); }
  else if (ref) {
    if (mark) {
      bw_put(&b, 1, 1);
      if (drop_st) { bw_ue(&b, 1); bw_ue(&b, 1); }
      bw_ue(&b, 4); bw_ue(&b, 1);
      bw_ue(&b, 3); bw_ue(&b, 0); bw_ue(&b, 0);
      bw_ue(&b, 0);
    } else bw_put(&b, 1, 0);
  }
  bw_se(&b, qp - 26);
  bw_ue(&b, 1);
  int skip_run = 0;
  for (int mby = r.row0; mby < r.row1; mby++)
    for (int mbx = r.x0; mbx < r.x1; mbx++) {
      const mb_t* m = &e->mbs[mby * e->mbw + mbx];
      if (!intra) {
        int sp[2];
        ltr_mv_pred_skip(e, mbx, mby, sp);
        if (m->type == 1 && m->i16_mode == 0 && m->cbp == 0 && m->mv[0] == sp[0] && m->mv[1] == sp[1]) { skip[mby * e->mbw + mbx] = 1; skip_run++; continue; }
        bw_ue(&b, skip_run); skip_run = 0;
      }
      if (m->type == 2) {
        bw_ue(&b, intra ? 25 : 30);
        if (b.nacc) bw_put(&b, 8 - b.nacc, 0);
        const uint8_t* ry = plane_y(e, e->cur); const uint8_t* ruv = plane_uv(e, e->cur);
        for (int y = 0; y < 16; y++) for (int x = 0; x < 16; x++) bw_put(&b, 8, ry[(size_t)(mby * 16 + y) * e->cw + mbx * 16 + x]);
        for (int k = 0; k < 2; k++)
          for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) bw_put(&b, 8, ruv[(size_t)(mby * 8 + y) * e->cw + (mbx * 8 + x) * 2 + k]);
        continue;
      }
      if (m->type == 3) {
        bw_ue(&b, intra ? 0 : 5);
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
        bw_ue(&b, intra ? t : t + 5);
        bw_ue(&b, m->chroma_mode);
        bw_se(&b, 0);
      } else {
        int mvp[2];
        ltr_mv_pred16(e, mbx, mby, m->i16_mode, mvp);
        bw_ue(&b, 0);
        if (active) bw_put(&b, 1, m->i16_mode ? 0 : 1);
        bw_se(&b, m->mv[0] - mvp[0]); bw_se(&b, m->mv[1] - mvp[1]);
        bw_ue(&b, cbp_to_codenum_inter[m->cbp]);
        if (m->cbp) bw_se(&b, 0);
      }
      write_residual(e, &b, skip, m, mbx, mby);
    }
  if (skip_run) bw_ue(&b, skip_run);
  *bits = (int64_t)bw_bits(&b);
  bw_trailing(&b);
  size_t n = nal_write(out, r.row0 == 0 && r.x0 == 0 && !idr, idr ? 3 : ref ? 2 : 0, idr ? 5 : 1, b.buf, b.pos);
  bw_free(&b);
  return n;
}

static void intra_picture(enc_t* e, const uint8_t* cur_nv12, int qp) {
  const int nsl = pic_n_slices(e);
#pragma omp parallel for schedule(dynamic, 1)
  for (int s = 0; s < nsl; s++) {
    const rect_t r = slice_rect(e, s);
    for (int mby = r.row0; mby < r.row1; mby++)
      for (int mbx = r.x0; mbx < r.x1; mbx++) encode_intra_mb(e, cur_nv12, mbx, mby, qp);
  }
}

static int64_t scut_encode(scut_t* sc, const uint8_t* cur_nv12, int idr, int rc_mode, int qp_fixed, int64_t target_bits, uint8_t* out) {
  ltr_t* l = sc->l;
  enc_t* e = l->e;
  layers_t* y = sc->y;
  const int mbs = e->mbw * e->mbh;
  /* the droppable layers (h264_layers_ref.c b2v_ref_layers_encode) */
  int is_ref = 1, ref_dist = 1;
  if (y) {
    if (idr) { y->since_idr = 0; y->frame_num = 0; }
    is_ref = idr || (y->since_idr & 1) == 0;
    ref_dist = y->last_was_ref ? 1 : 2;
    if (!y->last_was_ref) { uint8_t* t = e->recon[e->cur]; e->recon[e->cur] = y->spare; y->spare = t; }
    if (!idr && ref_dist != y->last_ref_dist)
      for (int i = 0; i < mbs; i++)
        if (e->mbs[i].type == 1) {
          e->mbs[i].mv[0] = (int16_t)scale_mv(e->mbs[i].mv[0], ref_dist, y->last_ref_dist);
          e->mbs[i].mv[1] = (int16_t)scale_mv(e->mbs[i].mv[1], ref_dist, y->last_ref_dist);
        }
    e->frame_num = y->frame_num;
  }
  /* h264_ltr_ref.c ltr_encode */
  const int k = (int)(e->pic & 1);
  const struct rcfb used = e->fb[k];
  const int qp = rc_frame_qp(e, &used, idr, rc_mode, qp_fixed, target_bits);
  e->cur ^= 1;
  e->pic_rows = idr ? 1 : e->slice_rows; e->pic_cols = idr ? e->seg_cols : e->mbw;
  if (idr) { e->frame_num = 0; }
  if (l->wide) {
    decimate(e, cur_nv12, dec_plane(l->w, e->recon[e->cur], 1));
    if (!idr) coarse_search(l->w, cur_nv12, qp);
  }
  const int active = !idr && l->lt_valid;
  int changed = mbs, mark = 0, cut = 0;
  int64_t c_intra = 0, c_inter = 0;
  if (idr) intra_picture(e, cur_nv12, qp);
  else {
    changed = 0;
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : changed)
    for (int mby = 0; mby < e->mbh; mby++)
      for (int mbx = 0; mbx < e->mbw; mbx++) {
        const int c = lean_class(l, cur_nv12, mbx, mby, qp);
        l->cls[mby * e->mbw + mbx] = (uint8_t)c;
        changed += c != LEAN_ZERO;
      }
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
    for (int pass = 0; pass < 2; pass++) {
#pragma omp parallel for schedule(dynamic, 1)
      for (int mby = 0; mby < e->mbh; mby++)
        for (int mbx = 0; mbx < e->mbw; mbx++)
          if (l->cls[mby * e->mbw + mbx] != LEAN_LT && is_anchor(e, mbx, mby) == (pass == 0)) ltr_inter_mb(l, cur_nv12, mbx, mby, qp);
    }
    if (sc->ltr_on) {
      const int lo = (mbs + LTR_CHANGED_MIN_DIV - 1) / LTR_CHANGED_MIN_DIV, hi = LTR_CHANGED_RATIO * l->prev_changed;
      mark = changed >= (lo > hi ? lo : hi);
    }
    /* the decision (h264_intra.cu k_scene_cut), then a cut picture coded again by the intra coder in the IDR grid */
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : c_intra, c_inter)
    for (int mby = 0; mby < e->mbh; mby++)
      for (int mbx = 0; mbx < e->mbw; mbx++) {
        c_intra += intra_cost(e, cur_nv12, mbx, mby, qp);
        c_inter += inter_cost(sc, cur_nv12, mbx, mby, qp, active);
      }
    cut = SCUT_INTRA_WEIGHT * c_intra < SCUT_INTER_WEIGHT * c_inter;
    if (cut) {
      e->pic_rows = 1; e->pic_cols = e->seg_cols;
      intra_picture(e, cur_nv12, qp);
    }
  }
  const int nsl = pic_n_slices(e);
  const int drop_st = mark && !active;
  uint8_t* skip = (uint8_t*)calloc(mbs, 1);
  const rect_t full = slice_rect(e, 0);
  const size_t per = (size_t)(full.row1 - full.row0) * (full.x1 - full.x0) * 1024 + 256;
  uint8_t* tmp = (uint8_t*)malloc(per * nsl);
  size_t* lens = (size_t*)calloc(nsl, sizeof(size_t));
  int64_t* sbits = (int64_t*)calloc(nsl, sizeof(int64_t));
#pragma omp parallel for schedule(dynamic, 1)
  for (int s = 0; s < nsl; s++) lens[s] = scut_code_slice(e, s, idr, idr || cut, is_ref, qp, active, mark, drop_st, skip, tmp + per * s, &sbits[s]);
  size_t o = 0; int64_t bits = 0;
  if (idr) { memcpy(out + o, e->sps, e->sps_len); o += e->sps_len; memcpy(out + o, e->pps, e->pps_len); o += e->pps_len; }
  for (int s = 0; s < nsl; s++) { memcpy(out + o, tmp + per * s, lens[s]); o += lens[s]; bits += sbits[s]; }
  free(tmp); free(lens); free(sbits);
  { int coded = 0; for (int i = 0; i < mbs; i++) coded |= !skip[i]; free(skip);
    struct rcfb init; memset(&init, 0, sizeof init); init.qp = -1;
    const struct rcfb prev = e->pic > 0 ? e->fb[k ^ 1] : init;
    rc_step(e, &e->fb[k], &prev, &used, bits + 40LL * nsl, qp, idr, coded, rc_mode, target_bits); }
  if (mark) { memcpy(l->lt, e->recon[e->cur ^ 1], (size_t)e->cw * e->ch * 3 / 2); l->lt_valid = 1; }
  if (idr) l->lt_valid = 0;
  l->prev_changed = changed;
  l->state[0] = active; l->state[1] = mark; l->state[2] = drop_st; l->state[3] = changed;
  sc->state[0] = cut; sc->state[1] = c_intra; sc->state[2] = c_inter; sc->state[3] = me_lambda[qp];
  e->last_qp = qp; e->last_bits = (int64_t)o * 8; e->pic++;
  if (idr) e->idr_count++;
  if (y) {
    if (!is_ref) { uint8_t* t = e->recon[e->cur ^ 1]; e->recon[e->cur ^ 1] = y->spare; y->spare = t; }
    else y->frame_num = (y->frame_num + 1) & 255;
    y->last_was_ref = is_ref; y->last_ref_dist = ref_dist;
    y->since_idr++;
  } else e->frame_num = (e->frame_num + 1) & 255;
  return (int64_t)o;
}

/* scene cuts on the encoder `h` (b2v_ref_enc_create, full frame), before its first picture.  ltr: the handle b2v_ref_ltr_create made on
 * `h` (the long-term reference on), or NULL (off); wide: wide-range motion; droppable: two temporal layers (not with ltr).  NULL in
 * striped mode.  Encode through b2v_ref_scut_encode from then on. */
void* b2v_ref_scut_create(void* h, void* ltr, int wide, int droppable) {
  enc_t* e = (enc_t*)h;
  if (e->stripe_rows || (ltr && droppable)) return NULL;
  scut_t* s = (scut_t*)calloc(1, sizeof *s);
  if (ltr) { s->l = (ltr_t*)ltr; s->ltr_on = 1; }
  else {
    uint8_t sps[64]; const int sps_len = e->sps_len;       /* the long-term layer's state without its SPS */
    memcpy(sps, e->sps, sizeof sps);
    s->l = (ltr_t*)scut_ltr_create_(h, wide);
    memcpy(e->sps, sps, sizeof sps); e->sps_len = sps_len;
    s->own_l = 1;
  }
  if (droppable) s->y = (layers_t*)scut_lyr_layers_create_(h);
  return s;
}
void b2v_ref_scut_destroy(void* sh) {
  scut_t* s = (scut_t*)sh;
  if (!s) return;
  if (s->own_l) scut_ltr_destroy_(s->l);
  scut_lyr_layers_destroy_(s->y);
  free(s);
}
int64_t b2v_ref_scut_encode(void* sh, const uint8_t* cur_nv12, int idr, int rc_mode, int qp_fixed, int64_t target_bits, uint8_t* out) {
  return scut_encode((scut_t*)sh, cur_nv12, idr, rc_mode, qp_fixed, target_bits, out);
}
/* the last picture: {cut, cost_intra, cost_inter, lambda} */
void b2v_ref_scut_state(void* sh, int64_t* out) { memcpy(out, ((scut_t*)sh)->state, sizeof ((scut_t*)sh)->state); }
