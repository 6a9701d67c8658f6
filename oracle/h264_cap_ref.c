/*
 * h264_cap_ref.c — CPU restatement of the picture size cap (B2V_FLAG_SIZE_CAP, include/b2video.h; DESIGN.md 5.15) on top of the
 * oracles of h264_ref.c, h264_layers_ref.c, h264_wide_ref.c, h264_ltr_ref.c and h264_scut_ref.c, all unchanged.  TEST INFRASTRUCTURE
 * ONLY.
 *
 * h264_scut_ref.c (and through it the other four) is compiled into this translation unit once more, every public name renamed below,
 * so that this file reaches the encoders' state and static helpers.  cap_encode is h264_scut_ref.c scut_encode with:
 *   - scene cuts optional;
 *   - the count (selkies_b200/csrc/h264_cap.cu k_size_cap): the bits of every coded macroblock's macroblock_layer() in a P picture,
 *     mb_type to its last residual block (an I_PCM macroblock: its mb_type and its 384 samples, not its alignment bits), summed;
 *     mb_skip_run and slice headers are not counted;
 *   - the rule: over the cap when ceil(bits / 8) > cap, then QP' = QP + d for the smallest d in 1..51-QP with
 *     bits <= (8 x cap x T[d]) >> 16, T[d] = round(65536 x 2^(d / 6)), or 51 when none qualifies;
 *   - the requantisation (h264_inter.cu k_requant): every macroblock coded again at QP' from the prediction its vector (or the
 *     long-term picture's zero vector) gives, by encode_inter_mb's residual coder, the I_PCM fallback decided again; then the slices
 *     at QP' (P_Skip decided again by the slice coder) and the rate-control step with QP'.
 * Full frame only, like h264_scut_ref.c.
 */
#define scut_lyr_enc_create_ cap_lyr_enc_create_
#define scut_lyr_enc_destroy_ cap_lyr_enc_destroy_
#define scut_lyr_enc_coded_w_ cap_lyr_enc_coded_w_
#define scut_lyr_enc_coded_h_ cap_lyr_enc_coded_h_
#define scut_lyr_enc_recon_ cap_lyr_enc_recon_
#define scut_lyr_enc_last_qp_ cap_lyr_enc_last_qp_
#define scut_lyr_enc_rc_state_ cap_lyr_enc_rc_state_
#define scut_lyr_enc_set_paintover_ cap_lyr_enc_set_paintover_
#define scut_lyr_enc_set_idr_slice_mbs_ cap_lyr_enc_set_idr_slice_mbs_
#define scut_lyr_enc_set_paintover_burst_ cap_lyr_enc_set_paintover_burst_
#define scut_lyr_enc_set_stripes_ cap_lyr_enc_set_stripes_
#define scut_lyr_enc_stripe_table_ cap_lyr_enc_stripe_table_
#define scut_lyr_enc_max_au_ cap_lyr_enc_max_au_
#define scut_lyr_enc_encode_ cap_lyr_enc_encode_
#define scut_lyr_layers_create_ cap_lyr_layers_create_
#define scut_lyr_layers_destroy_ cap_lyr_layers_destroy_
#define scut_lyr_layers_encode_ cap_lyr_layers_encode_
#define scut_wide_create_ cap_wide_create_
#define scut_wide_destroy_ cap_wide_destroy_
#define scut_wide_encode_ cap_wide_encode_
#define scut_wide_coarse_ cap_wide_coarse_
#define scut_wide_decimated_ cap_wide_decimated_
#define scut_ltr_create_ cap_ltr_create_
#define scut_ltr_destroy_ cap_ltr_destroy_
#define scut_ltr_encode_ cap_ltr_encode_
#define scut_ltr_state_ cap_ltr_state_
#define scut_ltr_picture_ cap_ltr_picture_
#define b2v_ref_scut_create cap_scut_create_
#define b2v_ref_scut_destroy cap_scut_destroy_
#define b2v_ref_scut_encode cap_scut_encode_
#define b2v_ref_scut_state cap_scut_state_
#include "h264_scut_ref.c"

/* T[d] = round(65536 x 2^(d / 6)) (selkies_b200/csrc/h264_common.cuh cap_t) */
static const int32_t CAP_T[52] = {
  65536, 73562, 82570, 92682, 104032, 116772, 131072, 147123, 165140, 185364, 208064, 233544, 262144, 294247, 330281, 370728,
  416128, 467088, 524288, 588493, 660561, 741455, 832255, 934175, 1048576, 1176987, 1321123, 1482910, 1664511, 1868350, 2097152,
  2353974, 2642246, 2965821, 3329021, 3736700, 4194304, 4707947, 5284492, 5931642, 6658043, 7473400, 8388608, 9415894, 10568984,
  11863283, 13316085, 14946800, 16777216, 18831788, 21137968, 23726566};

typedef struct {
  scut_t* s;
  int cut_on;
  int64_t state[4];        /* the last picture: recoded, the analysis's QP, the QP it was coded at, the count (0 for an IDR picture) */
} cap_t;

/* the count: macroblock_layer() bits of every coded macroblock of the P picture just analysed, pcm_alignment_zero_bit excepted, in
 * its P slice grid (the slice coder's order, so that P_Skip and nC see the same neighbours) */
static int64_t cap_count(enc_t* e, int active) {
  const int mbs = e->mbw * e->mbh, nsl = pic_n_slices(e);
  uint8_t* skip = (uint8_t*)calloc(mbs, 1);
  int64_t total = 0;
  for (int s = 0; s < nsl; s++) {
    const rect_t r = slice_rect(e, s);
    bitw_t b; bw_init(&b);
    for (int mby = r.row0; mby < r.row1; mby++)
      for (int mbx = r.x0; mbx < r.x1; mbx++) {
        const mb_t* m = &e->mbs[mby * e->mbw + mbx];
        int sp[2];
        ltr_mv_pred_skip(e, mbx, mby, sp);
        if (m->type == 1 && m->i16_mode == 0 && m->cbp == 0 && m->mv[0] == sp[0] && m->mv[1] == sp[1]) { skip[mby * e->mbw + mbx] = 1; continue; }
        const size_t p0 = bw_bits(&b);
        if (m->type == 2) { bw_ue(&b, 30); total += (int64_t)(bw_bits(&b) - p0) + 384 * 8; continue; }
        int mvp[2];
        ltr_mv_pred16(e, mbx, mby, m->i16_mode, mvp);
        bw_ue(&b, 0);
        if (active) bw_put(&b, 1, m->i16_mode ? 0 : 1);
        bw_se(&b, m->mv[0] - mvp[0]); bw_se(&b, m->mv[1] - mvp[1]);
        bw_ue(&b, cbp_to_codenum_inter[m->cbp]);
        if (m->cbp) bw_se(&b, 0);
        write_residual(e, &b, skip, m, mbx, mby);
        total += (int64_t)(bw_bits(&b) - p0);
      }
    bw_free(&b);
  }
  free(skip);
  return total;
}

/* the QP the picture is coded at: QP, or QP' when the count is over the cap */
static int cap_rule(int64_t bits, int qp, int cap_bytes) {
  if (cap_bytes <= 0 || qp >= 51 || (bits + 7) / 8 <= cap_bytes) return qp;
  int d = 1;
  while (d < 51 - qp && bits > ((int64_t)8 * cap_bytes * CAP_T[d]) >> 16) d++;
  return qp + d;
}

/* macroblock (mbx, mby) coded again at qp from its vector: the prediction (8.4.2.2, reference samples clamped to the picture), then
 * encode_inter_mb's residual coder, decimation included, and the I_PCM fallback with the picture's header budget */
static void requant_mb(ltr_t* l, const uint8_t* cur_nv12, int mbx, int mby, int qp) {
  enc_t* e = l->e;
  mb_t* m = &e->mbs[mby * e->mbw + mbx];
  const int lt = l->cls[mby * e->mbw + mbx] == LEAN_LT;
  const int mvx = lt ? 0 : m->me_mv[0], mvy = lt ? 0 : m->me_mv[1];
  const uint8_t* ref = lt ? l->lt : e->recon[e->cur ^ 1];
  const uint8_t* refuv = ref + (size_t)e->cw * e->ch;
  const int x0 = mbx * 16, y0 = mby * 16;
  uint8_t cy[256], cc[2][64], py[256], pc[2][64];
  load_cur(cur_nv12, e->cw, e->ch, mbx, mby, cy, cc);
  for (int r = 0; r < 16; r++)
    for (int c = 0; c < 16; c++) py[r * 16 + c] = (uint8_t)luma_sample(ref, e->cw, e->ch, x0 + c + (mvx >> 2), y0 + r + (mvy >> 2), mvx & 3, mvy & 3);
  const int xi = asr(mvx, 3), yi = asr(mvy, 3), xf = mvx & 7, yf = mvy & 7, cwc = e->cw / 2, chc = e->ch / 2;
  for (int r = 0; r < 8; r++)
    for (int c = 0; c < 8; c++) {
      const int xa = clip3(0, cwc - 1, mbx * 8 + xi + c), xb = clip3(0, cwc - 1, mbx * 8 + xi + c + 1);
      const int ya = clip3(0, chc - 1, mby * 8 + yi + r), yb = clip3(0, chc - 1, mby * 8 + yi + r + 1);
      for (int k = 0; k < 2; k++) {
        const int A = refuv[(size_t)ya * e->cw + xa * 2 + k], B = refuv[(size_t)ya * e->cw + xb * 2 + k];
        const int C = refuv[(size_t)yb * e->cw + xa * 2 + k], D = refuv[(size_t)yb * e->cw + xb * 2 + k];
        pc[k][r * 8 + c] = (uint8_t)(((8 - xf) * (8 - yf) * A + xf * (8 - yf) * B + (8 - xf) * yf * C + xf * yf * D + 32) >> 6);
      }
    }
  uint8_t* ry = plane_y(e, e->cur);
  int cbp = 0, score[16], s8[4] = {0, 0, 0, 0}, smb = 0;
  for (int b = 0; b < 16; b++) {
    const int bx = blk_x[b] * 4, by = blk_y[b] * 4;
    int res[16], dummy;
    for (int i = 0; i < 16; i++) { const int p = (by + (i >> 2)) * 16 + bx + (i & 3); res[i] = cy[p] - py[p]; }
    tq4x4(res, qp, 0, 0, m->coef[1 + b], &dummy);
    int sc = 0, zeros = 0, big = 0;
    for (int k = 0; k < 16; k++) {
      const int v = m->coef[1 + b][k];
      if (!v) { zeros++; continue; }
      if (iabs(v) > 1) big = 1;
      sc += zeros == 0 ? 3 : zeros <= 2 ? 2 : zeros <= 5 ? 1 : 0;
      zeros = 0;
    }
    score[b] = big ? 9 : sc;
    s8[b >> 2] += score[b]; smb += score[b];
  }
  for (int b = 0; b < 16; b++) {
    const int bx = blk_x[b] * 4, by = blk_y[b] * 4;
    if (s8[b >> 2] < 4 || smb < 6) memset(m->coef[1 + b], 0, sizeof m->coef[1 + b]);
    const int n = count_nz(m->coef[1 + b], 0, 16);
    m->nnz_l[blk_y[b] * 4 + blk_x[b]] = (uint8_t)n;
    if (n) cbp |= 1 << (b >> 2);
    int resid[16];
    recon4x4(m->coef[1 + b], qp, 0, 0, resid);
    for (int i = 0; i < 16; i++) {
      const int y = by + (i >> 2), x = bx + (i & 3);
      ry[(size_t)(y0 + y) * e->cw + x0 + x] = (uint8_t)clip1(py[y * 16 + x] + resid[i]);
    }
  }
  const int cbp_c = code_chroma(e, m, mbx, mby, qp, 0, cc, pc);
  m->type = 1; m->i16_mode = (int8_t)lt; m->cbp = (uint8_t)(cbp | (cbp_c << 4));
  m->mv[0] = (int16_t)mvx; m->mv[1] = (int16_t)mvy;
  if (l->wide) make_pcm_if_too_big_wide(e, m, cur_nv12, mbx, mby); else make_pcm_if_too_big(e, m, cur_nv12, mbx, mby);
}

static int64_t cap_encode(cap_t* cp, const uint8_t* cur_nv12, int idr, int rc_mode, int qp_fixed, int64_t target_bits, int cap_bytes, uint8_t* out) {
  scut_t* sc = cp->s;
  ltr_t* l = sc->l;
  enc_t* e = l->e;
  layers_t* y = sc->y;
  const int mbs = e->mbw * e->mbh;
  /* h264_scut_ref.c scut_encode, up to the decision */
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
  const int k = (int)(e->pic & 1);
  const struct rcfb used = e->fb[k];
  const int qp0 = rc_frame_qp(e, &used, idr, rc_mode, qp_fixed, target_bits);
  int qp = qp0;
  e->cur ^= 1;
  e->pic_rows = idr ? 1 : e->slice_rows; e->pic_cols = idr ? e->seg_cols : e->mbw;
  if (idr) { e->frame_num = 0; }
  if (l->wide) {
    decimate(e, cur_nv12, dec_plane(l->w, e->recon[e->cur], 1));
    if (!idr) coarse_search(l->w, cur_nv12, qp);
  }
  const int active = !idr && l->lt_valid;
  int changed = mbs, mark = 0, cut = 0;
  int64_t count = 0;
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
    if (cp->cut_on) {
      int64_t c_intra = 0, c_inter = 0;
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : c_intra, c_inter)
      for (int mby = 0; mby < e->mbh; mby++)
        for (int mbx = 0; mbx < e->mbw; mbx++) {
          c_intra += intra_cost(e, cur_nv12, mbx, mby, qp);
          c_inter += inter_cost(sc, cur_nv12, mbx, mby, qp, active);
        }
      cut = SCUT_INTRA_WEIGHT * c_intra < SCUT_INTER_WEIGHT * c_inter;
    }
    if (cut) {
      e->pic_rows = 1; e->pic_cols = e->seg_cols;
      intra_picture(e, cur_nv12, qp);
    } else {
      /* the count, the rule, the recode */
      count = cap_count(e, active);
      qp = cap_rule(count, qp0, cap_bytes);
      if (qp != qp0) {
#pragma omp parallel for schedule(dynamic, 1)
        for (int mby = 0; mby < e->mbh; mby++)
          for (int mbx = 0; mbx < e->mbw; mbx++) requant_mb(l, cur_nv12, mbx, mby, qp);
      }
    }
  }
  /* h264_scut_ref.c scut_encode from the slices on, at the final QP */
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
  sc->state[0] = cut;
  cp->state[0] = qp != qp0; cp->state[1] = qp0; cp->state[2] = qp; cp->state[3] = count;
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

/* the size cap on the encoder `h` (b2v_ref_enc_create, full frame), before its first picture; ltr, wide, droppable as for
 * b2v_ref_scut_create, scene_cut: scene cuts on or off.  NULL in striped mode.  Encode through b2v_ref_cap_encode from then on. */
void* b2v_ref_cap_create(void* h, void* ltr, int wide, int droppable, int scene_cut) {
  void* s = cap_scut_create_(h, ltr, wide, droppable);
  if (!s) return NULL;
  cap_t* c = (cap_t*)calloc(1, sizeof *c);
  c->s = (scut_t*)s; c->cut_on = scene_cut;
  return c;
}
void b2v_ref_cap_destroy(void* ch) {
  cap_t* c = (cap_t*)ch;
  if (!c) return;
  cap_scut_destroy_(c->s);
  free(c);
}
int64_t b2v_ref_cap_encode(void* ch, const uint8_t* cur_nv12, int idr, int rc_mode, int qp_fixed, int64_t target_bits, int cap_bytes, uint8_t* out) {
  return cap_encode((cap_t*)ch, cur_nv12, idr, rc_mode, qp_fixed, target_bits, cap_bytes, out);
}
/* the last picture: {recoded, QP of the analysis, QP it was coded at, the count in bits (0 for IDR and cut pictures)} */
void b2v_ref_cap_state(void* ch, int64_t* out) { memcpy(out, ((cap_t*)ch)->state, sizeof ((cap_t*)ch)->state); }
