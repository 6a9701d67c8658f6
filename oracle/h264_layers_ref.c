/*
 * h264_layers_ref.c — CPU restatement of droppable pictures (B2V_FLAG_DROPPABLE, include/b2video.h): two temporal layers on top of
 * the single-layer oracle of h264_ref.c, whose encoder runs unchanged for every picture.  TEST INFRASTRUCTURE ONLY.
 *
 * h264_ref.c is compiled into this translation unit a second time (its public names renamed below, its static helpers private to
 * this file), so that this file can reach the encoder's state; the handle it works on is one that b2v_ref_enc_create made (same
 * source, same layout).  Around each call of the single-layer encode it restates:
 *   - the layer rule: pictures are counted from each IDR (the IDR is 0); every P picture at an odd count is a non-reference picture;
 *   - reference selection: every P picture predicts from the last reference picture (one or two pictures back).  The encoder
 *     predicts from recon[cur] as it stands before the call and writes the other buffer; a third buffer (`spare`) holds the last
 *     reference picture's reconstruction while a non-reference picture is the last one, and is swapped in before the next picture.
 *     recon[cur] is the last coded picture after every call, droppable or not (b2v_ref_enc_recon);
 *   - predictor scaling: the previous picture's vectors (mbs[].mv, read only as the temporal predictor before the call overwrites
 *     them) are scaled by ref_dist / prev_ref_dist: doubled exactly, or halved rounding half away from zero,
 *     v -> sign(v) * ((|v| + 1) >> 1) (h264_inter.cu scale_mv);
 *   - the frame_num rule: it advances after reference pictures only (a non-reference picture carries the next reference's);
 *   - NAL and slice-header syntax of a non-reference picture: nal_ref_idc 0 and no dec_ref_pic_marking().  Its slices are coded
 *     again from the picture the single-layer encoder has just analysed (code_slice_nonref: h264_ref.c code_slice with that
 *     header; a header one bit shorter moves the I_PCM alignment, so the slices are re-coded, not edited);
 *   - the rate-control step of such a picture, run again from the same records on those slices' RBSP bits.
 * Full frame only: striped encoders are refused.
 */
#define b2v_ref_enc_create lyr_enc_create_
#define b2v_ref_enc_destroy lyr_enc_destroy_
#define b2v_ref_enc_coded_w lyr_enc_coded_w_
#define b2v_ref_enc_coded_h lyr_enc_coded_h_
#define b2v_ref_enc_recon lyr_enc_recon_
#define b2v_ref_enc_last_qp lyr_enc_last_qp_
#define b2v_ref_enc_rc_state lyr_enc_rc_state_
#define b2v_ref_enc_set_paintover lyr_enc_set_paintover_
#define b2v_ref_enc_set_idr_slice_mbs lyr_enc_set_idr_slice_mbs_
#define b2v_ref_enc_set_paintover_burst lyr_enc_set_paintover_burst_
#define b2v_ref_enc_set_stripes lyr_enc_set_stripes_
#define b2v_ref_enc_stripe_table lyr_enc_stripe_table_
#define b2v_ref_enc_max_au lyr_enc_max_au_
#define b2v_ref_enc_encode lyr_enc_encode_
#include "h264_ref.c"

typedef struct {
  enc_t* e;                /* the single-layer encoder (b2v_ref_enc_create) */
  uint8_t* spare;          /* the third reconstruction buffer */
  int64_t since_idr;       /* pictures since the last IDR */
  int last_was_ref, last_ref_dist, frame_num;
} layers_t;

static int scale_mv(int v, int num, int den) {
  if (num == den) return v;
  if (num > den) return 2 * v;
  return v < 0 ? -((-v + 1) >> 1) : (v + 1) >> 1;
}

/* 7.3.3 slice header of a P slice of a non-reference picture: write_slice_header without dec_ref_pic_marking() */
static void write_slice_header_nonref(bitw_t* b, int first_mb, int qp, int frame_num) {
  bw_ue(b, first_mb);
  bw_ue(b, 5);                                 /* slice_type P */
  bw_ue(b, 0);                                 /* pic_parameter_set_id */
  bw_put(b, 8, frame_num & 255);
  bw_put(b, 1, 0); bw_put(b, 1, 0);            /* num_ref_idx_active_override_flag, ref_pic_list_modification_flag_l0 */
  bw_se(b, qp - 26);                           /* slice_qp_delta */
  bw_ue(b, 1);                                 /* disable_deblocking_filter_idc */
}

/* code_slice of a P picture (full frame) as a slice of a non-reference picture: the same macroblock layer behind the header above,
 * nal_ref_idc 0.  Reads the picture the single-layer encoder has just analysed (its records and reconstruction). */
static size_t code_slice_nonref(enc_t* e, int s, int qp, int frame_num, uint8_t* skip, uint8_t* out, int64_t* bits) {
  bitw_t b; bw_init(&b);
  const rect_t r = slice_rect(e, s);
  write_slice_header_nonref(&b, r.row0 * e->mbw + r.x0, qp, frame_num);
  int skip_run = 0;
  for (int mby = r.row0; mby < r.row1; mby++)
    for (int mbx = r.x0; mbx < r.x1; mbx++) {
      const mb_t* m = &e->mbs[mby * e->mbw + mbx];
      int sp[2];
      mv_pred_skip(e, mbx, mby, sp);
      if (m->type == 1 && m->cbp == 0 && m->mv[0] == sp[0] && m->mv[1] == sp[1]) { skip[mby * e->mbw + mbx] = 1; skip_run++; continue; }
      bw_ue(&b, skip_run); skip_run = 0;
      if (m->type == 2) {                       /* I_PCM in a P slice */
        bw_ue(&b, 30);
        if (b.nacc) bw_put(&b, 8 - b.nacc, 0);
        const uint8_t* ry = plane_y(e, e->cur); const uint8_t* ruv = plane_uv(e, e->cur);
        for (int y = 0; y < 16; y++) for (int x = 0; x < 16; x++) bw_put(&b, 8, ry[(size_t)(mby * 16 + y) * e->cw + mbx * 16 + x]);
        for (int k = 0; k < 2; k++)
          for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) bw_put(&b, 8, ruv[(size_t)(mby * 8 + y) * e->cw + (mbx * 8 + x) * 2 + k]);
        continue;
      }
      if (m->type == 3) {                       /* I_NxN in a P slice */
        bw_ue(&b, 5);
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
        bw_ue(&b, t + 5);
        bw_ue(&b, m->chroma_mode);
        bw_se(&b, 0);
      } else {
        int mvp[2];
        mv_pred16(e, mbx, mby, mvp);
        bw_ue(&b, 0);                          /* P_L0_16x16 */
        bw_se(&b, m->mv[0] - mvp[0]); bw_se(&b, m->mv[1] - mvp[1]);
        bw_ue(&b, cbp_to_codenum_inter[m->cbp]);
        if (m->cbp) bw_se(&b, 0);
      }
      write_residual(e, &b, skip, m, mbx, mby);
    }
  if (skip_run) bw_ue(&b, skip_run);
  *bits = (int64_t)bw_bits(&b);
  bw_trailing(&b);
  size_t n = nal_write(out, r.row0 == 0 && r.x0 == 0, 0, 1, b.buf, b.pos);
  bw_free(&b);
  return n;
}

void* b2v_ref_layers_create(void* h) {
  enc_t* e = (enc_t*)h;
  if (e->stripe_rows) return NULL;
  layers_t* l = (layers_t*)calloc(1, sizeof *l);
  l->e = e;
  l->spare = (uint8_t*)calloc((size_t)e->cw * e->ch * 3 / 2, 1);
  l->last_was_ref = 1; l->last_ref_dist = 1;
  return l;
}
void b2v_ref_layers_destroy(void* lh) {
  layers_t* l = (layers_t*)lh;
  if (!l) return;
  free(l->spare); free(l);
}

/* b2v_ref_enc_encode of the encoder the layers were created on, with two temporal layers; returns the access unit's size */
int64_t b2v_ref_layers_encode(void* lh, const uint8_t* cur_nv12, int idr, int rc_mode, int qp_fixed, int64_t target_bits, uint8_t* out) {
  layers_t* l = (layers_t*)lh;
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
  int64_t n = lyr_enc_encode_(e, cur_nv12, idr, rc_mode, qp_fixed, target_bits, out);
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
