/*
 * oracle/h264_ref.c — CPU restatement of the H.264 Constrained-Baseline encoder stage.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under selkies_b200/ may link, import or execute this file;
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it.
 *
 * PARITY UNPINNED: the reference (selkies @1a9cd02b) contains no encoder.  Encoding happens in the
 * out-of-tree `pixelflux` wheel (pyproject.toml:37; media_pipeline.py:299-300) via libx264, or in
 * GStreamer x264enc in the legacy design (docs/component.md:322).  Neither is under /root/reference,
 * libx264 is not in this image, and the reference has no tests or golden bitstreams.  What the
 * reference does pin is the output FORMAT, and this file follows it:
 *   - Baseline/Constrained-Baseline, CAVLC, no B-frames, yuv420p, Annex-B, SPS/PPS in every IDR
 *     (src/selkies/webrtc/codecs/h264.py:281-321; rtc.py:394-401 sps-pps-idr-in-keyframe=1;
 *      webrtc/codecs/__init__.py:132-140 profile-level-id 42001f/42e01f)
 *   - splits cleanly on 00 00 01 (h264.py:238-263) => emulation prevention is mandatory
 * The algorithm restated is ITU-T H.264 (clauses cited inline) with this repo's own, documented
 * encoder decisions (DESIGN.md §5).  Independent pin: every stream this file produces is decoded by
 * libavcodec's h264 decoder (oracle/avdec.py) and must reproduce this encoder's reconstruction
 * bit-for-bit (tests/test_h264_oracle.py).
 *
 * Encoder decisions (the "spec" the CUDA path must match bit-for-bit):
 *   - one slice per `slice_rows` macroblock rows; deblocking disabled (disable_deblocking_filter_idc=1)
 *   - IDR pictures: per macroblock both Intra4x4 (9 modes, per block key = (SAD + lambda*(mode==predicted ? 1 : 4))*16
 *     + mode) and Intra16x16 are coded; the one with the smaller J = SSD + rd_lambda(qp) * luma bits is kept; I16 luma mode = argmin(SAD*4 + mode) over available modes
 *     {0 V, 1 H, 2 DC, 3 Plane}; chroma mode = argmin(SAD(Cb)+SAD(Cr))*4 + mode over {0 DC,1 H,2 V,3 Plane}
 *   - P pictures: every macroblock P_L0_16x16 (coded as P_Skip when mv == skip predictor and cbp == 0);
 *     full-pel exhaustive search dx in [-16,15], dy in [-16,16] against the previous reconstruction
 *     (coordinates clamped to the coded picture), cost = SAD + lambda(qp)*(bits_se(4dx)+bits_se(4dy)),
 *     argmin of (cost << 11 | (dy+16)*32 + (dx+16)); the search is skipped (mv = 0) when SAD(0,0) <= 96*lambda(qp);
 *     then half- and quarter-sample refinement (6-tap interpolation, 8 + 8 candidates) around the full-sample winner
 *   - quantisation: |l| = (|w|*MF + f) >> (15+qp/6), f = 2^(15+qp/6)/3 intra, /6 inter, |l| clamped to 2047
 *   - constant QP inside a picture; picture QP from the frame-level rate controller below.  The controller's feedback reaches
 *     the encoder TWO pictures late (picture k is coded with the controller state left by picture k-2): on the GPU the
 *     entropy coding of picture k-1 — where its size becomes known — overlaps the analysis of picture k (DESIGN.md §5.5/5.6)
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "h264_tables_ref.h"

/* ------------------------------------------------------------------ bit writer (7.2, 9.1) */
typedef struct { uint8_t* buf; size_t cap, pos; uint64_t acc; int nacc; } bitw_t;

static void bw_init(bitw_t* b) { b->cap = 1 << 16; b->buf = (uint8_t*)malloc(b->cap); b->pos = 0; b->acc = 0; b->nacc = 0; }
static void bw_free(bitw_t* b) { free(b->buf); b->buf = NULL; }
static void bw_byte(bitw_t* b, uint8_t v) {
  if (b->pos == b->cap) { b->cap *= 2; b->buf = (uint8_t*)realloc(b->buf, b->cap); }
  b->buf[b->pos++] = v;
}
static void bw_put(bitw_t* b, int n, uint32_t v) {   /* n <= 32, MSB first */
  if (n == 0) return;
  if (n < 32) v &= (1u << n) - 1;
  b->acc = (b->acc << n) | v;
  b->nacc += n;
  while (b->nacc >= 8) { bw_byte(b, (uint8_t)(b->acc >> (b->nacc - 8))); b->nacc -= 8; }
}
static void bw_ue(bitw_t* b, uint32_t v) {           /* 9.1 Exp-Golomb */
  uint32_t x = v + 1; int len = 0;
  while ((x >> len) > 1) len++;
  bw_put(b, len, 0);
  bw_put(b, len + 1, x);
}
static void bw_se(bitw_t* b, int v) { bw_ue(b, v > 0 ? (uint32_t)(2 * v - 1) : (uint32_t)(-2 * v)); }
static size_t bw_bits(const bitw_t* b) { return b->pos * 8 + b->nacc; }
static void bw_trailing(bitw_t* b) {                  /* 7.3.2.11 rbsp_trailing_bits */
  bw_put(b, 1, 1);
  if (b->nacc) bw_put(b, 8 - b->nacc, 0);
}

/* Annex B byte stream NAL unit with emulation prevention (7.4.1, B.1) */
static size_t nal_write(uint8_t* out, int long_start, int ref_idc, int type, const uint8_t* rbsp, size_t n) {
  size_t o = 0; int zeros = 0;
  if (long_start) out[o++] = 0;
  out[o++] = 0; out[o++] = 0; out[o++] = 1;
  out[o++] = (uint8_t)((ref_idc << 5) | type);
  for (size_t i = 0; i < n; i++) {
    if (zeros == 2 && rbsp[i] <= 3) { out[o++] = 3; zeros = 0; }
    out[o++] = rbsp[i];
    zeros = rbsp[i] == 0 ? zeros + 1 : 0;
  }
  return o;
}

/* ------------------------------------------------------------------ encoder state */
typedef struct {
  int16_t coef[27][16];   /* scan-order levels: 0 luma DC (I16x16), 1..16 luma blkIdx 0..15, 17/18 chroma DC Cb/Cr, 19..22 Cb AC, 23..26 Cr AC */
  uint8_t nnz_l[16];      /* TotalCoeff per luma 4x4 block, raster y*4+x */
  uint8_t nnz_c[2][4];    /* per chroma 4x4 block (AC), raster y*2+x */
  int8_t  type;           /* 0 I16x16, 1 P_L0_16x16, 2 I_PCM, 3 I_NxN (Intra4x4) */
  int8_t  i16_mode, chroma_mode;
  uint8_t cbp;            /* luma bits 0..3, chroma << 4 */
  int16_t mv[2];          /* quarter-sample units */
  int8_t  me_bad;         /* motion estimation found nothing better than a mean absolute difference of 32 per sample: new content */
  int16_t me_mv[2];       /* what motion estimation chose for this picture (== mv unless the macroblock then became I_PCM); read by the anchor predictor */
  int8_t  i4_modes[16];   /* Intra4x4PredMode per 4x4 block, raster y*4+x (type 3 only) */
} mb_t;

#define MAX_STRIPES 512
#define DEFAULT_SLICE_ROWS 8
typedef struct {
  int width, height, cw, ch, mbw, mbh, slice_rows, n_slices, auto_rows;
  /* IDR pictures may be cut finer than rows: slices of `seg_cols` macroblocks inside a row (whatever slice_rows is: that one governs P pictures).  The
   * macroblocks of an intra slice are a serial chain (left-neighbour prediction), so shorter slices = a shorter chain on the
   * GPU (DESIGN.md §5.2).  pic_seg is the value in force for the picture being coded (0 = whole rows). */
  int seg_cols, pic_seg;
  uint8_t* recon[2];      /* NV12, coded size; recon[cur] is being written, recon[cur^1] is the reference */
  int cur;
  mb_t* mbs;
  int frame_num, idr_count;
  /* rate controller / paint-over scheduler: fb[k & 1] is the feedback record written after picture k; picture k is coded from
   * fb[k & 1] as it stood BEFORE that, i.e. the state after picture k-2 (see rc_step) */
  struct rcfb { int32_t qp, static_run, remaining, paint, debt; int64_t fullness, X; } fb[2];
  int64_t pic;            /* pictures encoded so far */
  int paint_trigger, paint_qp, paint_burst;   /* paint-over: `paint_burst` finer pictures after `paint_trigger` all-skipped pictures */
  int last_qp; int64_t last_bits;
  uint8_t sps[64], pps[32]; int sps_len, pps_len;
  /* striped mode (pixelflux h264_fullframe = False): the picture is cut into bands of stripe_rows macroblock rows, each an
   * independent H.264 stream (own SPS, own frame_num, motion vectors confined to the band by reference-sample clamping) */
  int stripe_rows, n_stripes;
  int stripe_fn[MAX_STRIPES];
  int32_t stripe_tab[MAX_STRIPES][3];   /* last picture: byte offset, size, coded flag */
  uint8_t sps_band[2][64]; int sps_band_len[2];   /* [0] regular band, [1] last band (may be shorter / cropped) */
  int no_i4, no_tpred, no_refine_cap, no_anchor, no_newcontent, no_zcand;    /* A/B switches for experiments (environment B2V_REF_NO_I4 / B2V_REF_NO_TPRED / B2V_REF_NO_REFINE_CAP, read once at create) */
} enc_t;

static int clip3(int lo, int hi, int v) { return v < lo ? lo : (v > hi ? hi : v); }
static int clip1(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }
static int iabs(int v) { return v < 0 ? -v : v; }
static int asr(int v, int s) { return v >= 0 ? (v >> s) : -((-v + (1 << s) - 1) >> s); }

static int level_idc_for(int mbs) { return mbs <= 3600 ? 31 : mbs <= 8704 ? 42 : mbs <= 22080 ? 51 : mbs <= 36864 ? 52 : 62; }

/* 7.3.2.1 SPS, 7.3.2.2 PPS */
static int build_sps(uint8_t* dst, int mbw, int mbh, int crop_r, int crop_b) {
  bitw_t b; bw_init(&b);
  bw_put(&b, 8, 66);            /* profile_idc Baseline */
  bw_put(&b, 8, 0xC0);          /* constraint_set0_flag, constraint_set1_flag => Constrained Baseline */
  bw_put(&b, 8, level_idc_for(mbw * mbh));
  bw_ue(&b, 0);                 /* seq_parameter_set_id */
  bw_ue(&b, 4);                 /* log2_max_frame_num_minus4 => frame_num is 8 bits */
  bw_ue(&b, 2);                 /* pic_order_cnt_type 2: output order == decoding order */
  bw_ue(&b, 1);                 /* max_num_ref_frames */
  bw_put(&b, 1, 0);             /* gaps_in_frame_num_value_allowed_flag */
  bw_ue(&b, mbw - 1);
  bw_ue(&b, mbh - 1);
  bw_put(&b, 1, 1);             /* frame_mbs_only_flag */
  bw_put(&b, 1, 1);             /* direct_8x8_inference_flag */
  if (crop_r || crop_b) { bw_put(&b, 1, 1); bw_ue(&b, 0); bw_ue(&b, crop_r); bw_ue(&b, 0); bw_ue(&b, crop_b); }
  else bw_put(&b, 1, 0);
  /* E.1.1 VUI: colour description (the CSC stage is BT.709 limited range, centre-sited chroma) and a
   * bitstream restriction telling decoders there is no reordering (low-latency output) */
  bw_put(&b, 1, 1);             /* vui_parameters_present_flag */
  bw_put(&b, 1, 0);             /* aspect_ratio_info_present_flag */
  bw_put(&b, 1, 0);             /* overscan_info_present_flag */
  bw_put(&b, 1, 1);             /* video_signal_type_present_flag */
  bw_put(&b, 3, 5);             /* video_format: unspecified */
  bw_put(&b, 1, 0);             /* video_full_range_flag: limited */
  bw_put(&b, 1, 1);             /* colour_description_present_flag */
  bw_put(&b, 8, 1); bw_put(&b, 8, 1); bw_put(&b, 8, 1);   /* primaries / transfer / matrix = BT.709 */
  bw_put(&b, 1, 1);             /* chroma_loc_info_present_flag */
  bw_ue(&b, 1); bw_ue(&b, 1);   /* chroma_sample_loc_type top/bottom = 1 (centre) */
  bw_put(&b, 1, 0);             /* timing_info_present_flag */
  bw_put(&b, 1, 0);             /* nal_hrd_parameters_present_flag */
  bw_put(&b, 1, 0);             /* vcl_hrd_parameters_present_flag */
  bw_put(&b, 1, 0);             /* pic_struct_present_flag */
  bw_put(&b, 1, 1);             /* bitstream_restriction_flag */
  bw_put(&b, 1, 1);             /* motion_vectors_over_pic_boundaries_flag */
  bw_ue(&b, 0); bw_ue(&b, 0);   /* max_bytes_per_pic_denom, max_bits_per_mb_denom */
  bw_ue(&b, 10); bw_ue(&b, 10); /* log2_max_mv_length_horizontal / vertical */
  bw_ue(&b, 0);                 /* max_num_reorder_frames */
  bw_ue(&b, 1);                 /* max_dec_frame_buffering */
  bw_trailing(&b);
  int n = (int)nal_write(dst, 1, 3, 7, b.buf, b.pos);
  bw_free(&b);
  return n;
}
static void write_param_sets(enc_t* e) {
  bitw_t b;
  e->sps_len = build_sps(e->sps, e->mbw, e->mbh, (e->cw - e->width) / 2, (e->ch - e->height) / 2);
  bw_init(&b);
  bw_ue(&b, 0); bw_ue(&b, 0);   /* pps id, sps id */
  bw_put(&b, 1, 0);             /* entropy_coding_mode_flag: CAVLC */
  bw_put(&b, 1, 0);             /* bottom_field_pic_order_in_frame_present_flag */
  bw_ue(&b, 0);                 /* num_slice_groups_minus1 */
  bw_ue(&b, 0); bw_ue(&b, 0);   /* num_ref_idx_l0/l1_default_active_minus1 */
  bw_put(&b, 1, 0);             /* weighted_pred_flag */
  bw_put(&b, 2, 0);             /* weighted_bipred_idc */
  bw_se(&b, 0); bw_se(&b, 0);   /* pic_init_qp_minus26, pic_init_qs_minus26 */
  bw_se(&b, 0);                 /* chroma_qp_index_offset */
  bw_put(&b, 1, 1);             /* deblocking_filter_control_present_flag */
  bw_put(&b, 1, 0);             /* constrained_intra_pred_flag */
  bw_put(&b, 1, 0);             /* redundant_pic_cnt_present_flag */
  bw_trailing(&b);
  e->pps_len = (int)nal_write(e->pps, 1, 3, 8, b.buf, b.pos);
  bw_free(&b);
}

/* ------------------------------------------------------------------ transforms (8.5) */
static int pos_class(int raster) { int x = raster & 3, y = raster >> 2; return ((x | y) & 1) == 0 ? 0 : ((x & y) & 1) ? 1 : 2; }

static void fwd4x4(const int in[16], int out[16]) {      /* W = Cf X Cf^T, rows then columns */
  int t[16];
  for (int i = 0; i < 4; i++) {
    const int* r = in + 4 * i;
    int s03 = r[0] + r[3], d03 = r[0] - r[3], s12 = r[1] + r[2], d12 = r[1] - r[2];
    t[4 * i + 0] = s03 + s12; t[4 * i + 1] = 2 * d03 + d12; t[4 * i + 2] = s03 - s12; t[4 * i + 3] = d03 - 2 * d12;
  }
  for (int j = 0; j < 4; j++) {
    int s03 = t[j] + t[12 + j], d03 = t[j] - t[12 + j], s12 = t[4 + j] + t[8 + j], d12 = t[4 + j] - t[8 + j];
    out[j] = s03 + s12; out[4 + j] = 2 * d03 + d12; out[8 + j] = s03 - s12; out[12 + j] = d03 - 2 * d12;
  }
}
static void inv4x4(const int d[16], int r[16]) {         /* 8.5.12.2: rows, then columns, (x+32)>>6 */
  int t[16];
  for (int i = 0; i < 4; i++) {
    const int* p = d + 4 * i;
    int e0 = p[0] + p[2], e1 = p[0] - p[2], e2 = (p[1] >> 1) - p[3], e3 = p[1] + (p[3] >> 1);
    t[4 * i + 0] = e0 + e3; t[4 * i + 1] = e1 + e2; t[4 * i + 2] = e1 - e2; t[4 * i + 3] = e0 - e3;
  }
  for (int j = 0; j < 4; j++) {
    int e0 = t[j] + t[8 + j], e1 = t[j] - t[8 + j], e2 = (t[4 + j] >> 1) - t[12 + j], e3 = t[4 + j] + (t[12 + j] >> 1);
    r[j] = (e0 + e3 + 32) >> 6; r[4 + j] = (e1 + e2 + 32) >> 6; r[8 + j] = (e1 - e2 + 32) >> 6; r[12 + j] = (e0 - e3 + 32) >> 6;
  }
}
static void hadamard4x4(const int in[16], int out[16]) { /* H X H, H symmetric */
  int t[16];
  for (int i = 0; i < 4; i++) {
    const int* r = in + 4 * i;
    int s01 = r[0] + r[1], d01 = r[0] - r[1], s23 = r[2] + r[3], d23 = r[2] - r[3];
    t[4 * i + 0] = s01 + s23; t[4 * i + 1] = s01 - s23; t[4 * i + 2] = d01 - d23; t[4 * i + 3] = d01 + d23;
  }
  for (int j = 0; j < 4; j++) {
    int s01 = t[j] + t[4 + j], d01 = t[j] - t[4 + j], s23 = t[8 + j] + t[12 + j], d23 = t[8 + j] - t[12 + j];
    out[j] = s01 + s23; out[4 + j] = s01 - s23; out[8 + j] = d01 - d23; out[12 + j] = d01 + d23;
  }
}
static int quant1(int w, int mf, int f, int qbits) {
  int a = (iabs(w) * mf + f) >> qbits;
  if (a > 2047) a = 2047;
  return w < 0 ? -a : a;
}

/* Transform + quantise + reconstruct one 4x4 block of residual `res` (raster).
 * levels_scan: 16 scan-order levels out (position 0 left 0 when dc_separate).
 * dc_separate: the DC coefficient is handled by the caller (Intra16x16 / chroma): w_dc receives the
 * forward DC; the block is reconstructed later by recon4x4() once the dequantised DC is known. */
static void tq4x4(const int res[16], int qp, int intra, int dc_separate, int16_t levels_scan[16], int* w_dc) {
  int w[16];
  fwd4x4(res, w);
  int qbits = 15 + qp / 6, f = (1 << qbits) / (intra ? 3 : 6);
  for (int k = 0; k < 16; k++) {
    int r = zigzag4x4[k];
    if (k == 0 && dc_separate) { *w_dc = w[0]; levels_scan[0] = 0; continue; }
    levels_scan[k] = (int16_t)quant1(w[r], quant_mf[qp % 6][pos_class(r)], f, qbits);
  }
}
/* dequantise (8.5.12.1) + inverse transform; dc_value (already dequantised) replaces d[0] when use_dc */
static void recon4x4(const int16_t levels_scan[16], int qp, int use_dc, int dc_value, int resid[16]) {
  int d[16];
  for (int k = 0; k < 16; k++) {
    int r = zigzag4x4[k];
    d[r] = (levels_scan[k] * dequant_v[qp % 6][pos_class(r)]) << (qp / 6);
  }
  if (use_dc) d[0] = dc_value;
  inv4x4(d, resid);
}
static int count_nz(const int16_t* l, int from, int to) { int n = 0; for (int k = from; k < to; k++) n += l[k] != 0; return n; }

/* ------------------------------------------------------------------ frame access helpers */
static uint8_t* plane_y(enc_t* e, int idx) { return e->recon[idx]; }
static uint8_t* plane_uv(enc_t* e, int idx) { return e->recon[idx] + (size_t)e->cw * e->ch; }

static int slice_first_row(const enc_t* e, int mby) { return (mby / e->slice_rows) * e->slice_rows; }
static int avail_top(const enc_t* e, int mby) { return e->pic_seg ? 0 : mby > slice_first_row(e, mby); }
static int avail_left(const enc_t* e, int mbx) { return e->pic_seg ? (mbx % e->pic_seg) != 0 : mbx > 0; }
static int pic_segs(const enc_t* e) { return e->pic_seg ? (e->mbw + e->pic_seg - 1) / e->pic_seg : 1; }
static int pic_n_slices(const enc_t* e) { return e->pic_seg ? e->mbh * pic_segs(e) : e->n_slices; }
/* default IDR slicing: about 540 slices per picture, none shorter than 30 macroblocks */
static int auto_seg_cols(int mbw, int mbh) {
  int segs = 540 / mbh, cap = mbw / 30;
  if (segs > cap) segs = cap;
  if (segs <= 1) return mbw;          /* one slice per macroblock row */
  return (mbw + segs - 1) / segs;
}
static void make_pcm_if_too_big(enc_t* e, mb_t* m, const uint8_t* cur_nv12, int mbx, int mby);   /* defined after the CAVLC coder */
static void cavlc_block(bitw_t* b, const int16_t* lv, int start, int maxc, int nC);

/* ------------------------------------------------------------------ chroma: shared by I and P macroblocks */
/* cur/pred: [2][64] raster 8x8 per component.  Writes levels, nnz_c, chroma cbp; reconstructs into the frame. */
static int code_chroma(enc_t* e, mb_t* m, int mbx, int mby, int qp, int intra, const uint8_t cur[2][64], const uint8_t pred[2][64]) {
  int qpc = chroma_qp_tab[clip3(0, 51, qp)];
  int any_dc = 0, any_ac = 0;
  uint8_t* uv = plane_uv(e, e->cur);
  for (int c = 0; c < 2; c++) {
    int dcs[4];
    for (int b = 0; b < 4; b++) {
      int bx = (b & 1) * 4, by = (b >> 1) * 4, res[16];
      for (int i = 0; i < 16; i++) { int p = (by + (i >> 2)) * 8 + bx + (i & 3); res[i] = cur[c][p] - pred[c][p]; }
      tq4x4(res, qpc, intra, 1, m->coef[19 + c * 4 + b], &dcs[b]);
      m->nnz_c[c][b] = (uint8_t)count_nz(m->coef[19 + c * 4 + b], 1, 16);
      any_ac |= m->nnz_c[c][b];
    }
    /* 2x2 DC: forward Hadamard, quantise with doubled dead zone and one more shift */
    int t[4] = { dcs[0] + dcs[1] + dcs[2] + dcs[3], dcs[0] - dcs[1] + dcs[2] - dcs[3], dcs[0] + dcs[1] - dcs[2] - dcs[3], dcs[0] - dcs[1] - dcs[2] + dcs[3] };
    int qbits = 15 + qpc / 6, f = (1 << qbits) / (intra ? 3 : 6);
    int16_t* dl = m->coef[17 + c];
    for (int k = 0; k < 4; k++) { dl[k] = (int16_t)quant1(t[k], quant_mf[qpc % 6][0], 2 * f, qbits + 1); any_dc |= dl[k] != 0; }
    for (int k = 4; k < 16; k++) dl[k] = 0;
    /* 8.5.11.1/2: inverse 2x2 + chroma DC dequant */
    int fq[4] = { dl[0] + dl[1] + dl[2] + dl[3], dl[0] - dl[1] + dl[2] - dl[3], dl[0] + dl[1] - dl[2] - dl[3], dl[0] - dl[1] - dl[2] + dl[3] };
    int ls = 16 * dequant_v[qpc % 6][0];
    for (int b = 0; b < 4; b++) {
      int dc = ((fq[b] * ls) << (qpc / 6)) >> 5;
      int resid[16];
      recon4x4(m->coef[19 + c * 4 + b], qpc, 1, dc, resid);
      int bx = (b & 1) * 4, by = (b >> 1) * 4;
      for (int i = 0; i < 16; i++) {
        int y = by + (i >> 2), x = bx + (i & 3);
        uv[(size_t)(mby * 8 + y) * e->cw + (mbx * 8 + x) * 2 + c] = (uint8_t)clip1(pred[c][y * 8 + x] + resid[i]);
      }
    }
  }
  return any_ac ? 2 : (any_dc ? 1 : 0);
}

static void load_cur(const uint8_t* nv12, int cw, int ch, int mbx, int mby, uint8_t y[256], uint8_t c[2][64]) {
  for (int r = 0; r < 16; r++) memcpy(y + 16 * r, nv12 + (size_t)(mby * 16 + r) * cw + mbx * 16, 16);
  const uint8_t* uv = nv12 + (size_t)cw * ch;
  for (int r = 0; r < 8; r++)
    for (int x = 0; x < 8; x++) {
      c[0][r * 8 + x] = uv[(size_t)(mby * 8 + r) * cw + (mbx * 8 + x) * 2];
      c[1][r * 8 + x] = uv[(size_t)(mby * 8 + r) * cw + (mbx * 8 + x) * 2 + 1];
    }
}

/* ------------------------------------------------------------------ intra macroblock (8.3.3, 8.3.4) */
static void pred16(int mode, const uint8_t* top, const uint8_t* left, int tl, int has_top, int has_left, uint8_t out[256]) {
  if (mode == 0) { for (int y = 0; y < 16; y++) memcpy(out + 16 * y, top, 16); }
  else if (mode == 1) { for (int y = 0; y < 16; y++) memset(out + 16 * y, left[y], 16); }
  else if (mode == 2) {
    int s = 0, dc;
    if (has_top) for (int i = 0; i < 16; i++) s += top[i];
    if (has_left) for (int i = 0; i < 16; i++) s += left[i];
    dc = has_top && has_left ? (s + 16) >> 5 : (has_top || has_left) ? (s + 8) >> 4 : 128;
    memset(out, dc, 256);
  } else {
    int H = 0, V = 0;
    for (int i = 0; i < 8; i++) {
      H += (i + 1) * (top[8 + i] - (i == 7 ? tl : top[6 - i]));
      V += (i + 1) * (left[8 + i] - (i == 7 ? tl : left[6 - i]));
    }
    int a = 16 * (left[15] + top[15]), b = asr(5 * H + 32, 6), c = asr(5 * V + 32, 6);
    for (int y = 0; y < 16; y++)
      for (int x = 0; x < 16; x++) out[16 * y + x] = (uint8_t)clip1(asr(a + b * (x - 7) + c * (y - 7) + 16, 5));
  }
}
static void pred8c(int mode, const uint8_t* top, const uint8_t* left, int tl, int has_top, int has_left, uint8_t out[64]) {
  if (mode == 2) { for (int y = 0; y < 8; y++) memcpy(out + 8 * y, top, 8); }
  else if (mode == 1) { for (int y = 0; y < 8; y++) memset(out + 8 * y, left[y], 8); }
  else if (mode == 0) {
    for (int b = 0; b < 4; b++) {
      int bx = (b & 1) * 4, by = (b >> 1) * 4, st = 0, sl = 0, dc;
      for (int i = 0; i < 4; i++) { if (has_top) st += top[bx + i]; if (has_left) sl += left[by + i]; }
      if (b == 0 || b == 3) dc = has_top && has_left ? (st + sl + 4) >> 3 : has_top ? (st + 2) >> 2 : has_left ? (sl + 2) >> 2 : 128;
      else if (b == 1) dc = has_top ? (st + 2) >> 2 : has_left ? (sl + 2) >> 2 : 128;
      else dc = has_left ? (sl + 2) >> 2 : has_top ? (st + 2) >> 2 : 128;
      for (int y = 0; y < 4; y++) memset(out + 8 * (by + y) + bx, dc, 4);
    }
  } else {
    int H = 0, V = 0;
    for (int i = 0; i < 4; i++) {
      H += (i + 1) * (top[4 + i] - (i == 3 ? tl : top[2 - i]));
      V += (i + 1) * (left[4 + i] - (i == 3 ? tl : left[2 - i]));
    }
    int a = 16 * (left[7] + top[7]), b = asr(34 * H + 32, 6), c = asr(34 * V + 32, 6);
    for (int y = 0; y < 8; y++)
      for (int x = 0; x < 8; x++) out[8 * y + x] = (uint8_t)clip1(asr(a + b * (x - 3) + c * (y - 3) + 16, 5));
  }
}
static int sad_n(const uint8_t* a, const uint8_t* b, int n) { int s = 0; for (int i = 0; i < n; i++) s += iabs(a[i] - b[i]); return s; }


#define I4_SKIP_SAD_PER_LAMBDA 32   /* Intra4x4 is only tried when the best Intra16x16 SAD exceeds 32*lambda */
/* ------------------------------------------------------------------ Intra4x4 (8.3.1) */
/* e[0..3] = left samples bottom..top (l3,l2,l1,l0), e[4] = top-left M, e[5..12] = top samples t0..t7 (t4..t7 = top-right) */
static int f3(int a, int b, int c) { return (a + 2 * b + c + 2) >> 2; }
static int f2(int a, int b) { return (a + b + 1) >> 1; }
static int pred4_pixel(int mode, int x, int y, const uint8_t* e, int has_a, int has_b) {
  const uint8_t* t = e + 5; /* t[-1] = M */
#define L(i) ((i) < 0 ? e[4] : e[3 - (i)])
  switch (mode) {
    case 0: return t[x];
    case 1: return L(y);
    case 2: {
      int s = 0;
      if (has_a && has_b) { for (int i = 0; i < 4; i++) s += t[i] + L(i); return (s + 4) >> 3; }
      if (has_b) { for (int i = 0; i < 4; i++) s += t[i]; return (s + 2) >> 2; }
      if (has_a) { for (int i = 0; i < 4; i++) s += L(i); return (s + 2) >> 2; }
      return 128;
    }
    case 3: return (x == 3 && y == 3) ? (t[6] + 3 * t[7] + 2) >> 2 : f3(t[x + y], t[x + y + 1], t[x + y + 2]);
    case 4: return f3(e[4 + x - y - 1], e[4 + x - y], e[4 + x - y + 1]);
    case 5: {
      int z = 2 * x - y;
      if (z >= 0 && !(z & 1)) return f2(t[x - (y >> 1) - 1], t[x - (y >> 1)]);
      if (z >= 0) return f3(t[x - (y >> 1) - 2], t[x - (y >> 1) - 1], t[x - (y >> 1)]);
      if (z == -1) return f3(L(0), e[4], t[0]);
      return f3(L(y - 1), L(y - 2), L(y - 3));
    }
    case 6: {
      int z = 2 * y - x;
      if (z >= 0 && !(z & 1)) return f2(L(y - (x >> 1) - 1), L(y - (x >> 1)));
      if (z >= 0) return f3(L(y - (x >> 1) - 2), L(y - (x >> 1) - 1), L(y - (x >> 1)));
      if (z == -1) return f3(L(0), e[4], t[0]);
      return f3(t[x - 1], t[x - 2], t[x - 3]);
    }
    case 7: return (y & 1) ? f3(t[x + (y >> 1)], t[x + (y >> 1) + 1], t[x + (y >> 1) + 2]) : f2(t[x + (y >> 1)], t[x + (y >> 1) + 1]);
    default: {
      int z = x + 2 * y;
      if (z > 5) return L(3);
      if (z == 5) return (L(2) + 3 * L(3) + 2) >> 2;
      if (z & 1) return f3(L(y + (x >> 1)), L(y + (x >> 1) + 1), L(y + (x >> 1) + 2));
      return f2(L(y + (x >> 1)), L(y + (x >> 1) + 1));
    }
  }
#undef L
}
static int i4_mode_ok(int mode, int has_a, int has_b, int has_d) {
  switch (mode) {
    case 0: case 3: case 7: return has_b;
    case 1: case 8: return has_a;
    case 2: return 1;
    default: return has_a && has_b && has_d;
  }
}
/* predIntra4x4PredMode (8.3.1.1) for block (bx,by) of macroblock (mbx,mby) */
static int i4_pred_mode(const enc_t* e, int mbx, int mby, int bx, int by) {
  const mb_t* m = &e->mbs[mby * e->mbw + mbx];
  int ma, mb_;
  if (bx > 0) ma = m->i4_modes[by * 4 + bx - 1];
  else { if (!avail_left(e, mbx)) return 2; const mb_t* n = m - 1; ma = n->type == 3 ? n->i4_modes[by * 4 + 3] : 2; }
  if (by > 0) mb_ = m->i4_modes[(by - 1) * 4 + bx];
  else { if (!avail_top(e, mby)) return 2; const mb_t* n = m - e->mbw; mb_ = n->type == 3 ? n->i4_modes[12 + bx] : 2; }
  return ma < mb_ ? ma : mb_;
}
/* C (top-right) availability of block (bx,by) inside the macroblock: decoded earlier in blkIdx order */
static const uint8_t i4_tr_inside[16] = { 2,2,2,3, 1,0,1,0, 1,1,1,0, 1,0,1,0 };   /* raster; row 0: 2 = from the MB above, 3 = from the MB above-right */

/* Code the luma of one macroblock as 16 Intra4x4 blocks in decoding order (reconstruction is written to the frame
 * because each block predicts from its already reconstructed neighbours).  Returns sum(SAD + lambda*mode bits). */
static int intra4x4_pass(enc_t* e, mb_t* m, const uint8_t cy[256], int mbx, int mby, int qp) {
  uint8_t* ry = plane_y(e, e->cur);
  const int x0 = mbx * 16, y0 = mby * 16, lambda = me_lambda[qp];
  const int mb_left = avail_left(e, mbx), mb_top = avail_top(e, mby), mb_tr = mb_top && mbx + 1 < e->mbw;
  int cost = 0;
  for (int blk = 0; blk < 16; blk++) {
    const int bx = blk_x[blk], by = blk_y[blk], px = x0 + bx * 4, py = y0 + by * 4;
    const int has_a = bx > 0 || mb_left, has_b = by > 0 || mb_top;
    const int has_d = (bx > 0 && by > 0) ? 1 : (bx > 0) ? mb_top : (by > 0) ? mb_left : (mb_left && mb_top);
    const int trc = i4_tr_inside[by * 4 + bx];
    const int has_c = trc == 1 ? 1 : trc == 2 ? mb_top : trc == 3 ? mb_tr : 0;
    uint8_t ed[13];
    memset(ed, 128, sizeof ed);
    if (has_a) for (int i = 0; i < 4; i++) ed[3 - i] = ry[(size_t)(py + i) * e->cw + px - 1];
    if (has_d) ed[4] = ry[(size_t)(py - 1) * e->cw + px - 1];
    if (has_b) {
      for (int i = 0; i < 4; i++) ed[5 + i] = ry[(size_t)(py - 1) * e->cw + px + i];
      for (int i = 4; i < 8; i++) ed[5 + i] = has_c ? ry[(size_t)(py - 1) * e->cw + px + i] : ed[8];   /* 8.3.1.2: replicate p[3,-1] */
    }
    const int pm = i4_pred_mode(e, mbx, mby, bx, by);
    int best_key = 1 << 30, best_mode = 2; uint8_t best_pred[16];
    for (int mode = 0; mode < 9; mode++) {
      if (!i4_mode_ok(mode, has_a, has_b, has_d)) continue;
      uint8_t pr[16]; int sad = 0;
      for (int i = 0; i < 16; i++) { pr[i] = (uint8_t)pred4_pixel(mode, i & 3, i >> 2, ed, has_a, has_b); sad += iabs(cy[(by * 4 + (i >> 2)) * 16 + bx * 4 + (i & 3)] - pr[i]); }
      int key = (sad + lambda * (mode == pm ? 1 : 4)) * 16 + mode;
      if (key < best_key) { best_key = key; best_mode = mode; memcpy(best_pred, pr, 16); }
    }
    m->i4_modes[by * 4 + bx] = (int8_t)best_mode;
    cost += best_key >> 4;
    int res[16], dummy, resid[16];
    for (int i = 0; i < 16; i++) res[i] = cy[(by * 4 + (i >> 2)) * 16 + bx * 4 + (i & 3)] - best_pred[i];
    tq4x4(res, qp, 1, 0, m->coef[1 + blk], &dummy);
    m->nnz_l[by * 4 + bx] = (uint8_t)count_nz(m->coef[1 + blk], 0, 16);
    recon4x4(m->coef[1 + blk], qp, 0, 0, resid);
    for (int i = 0; i < 16; i++) ry[(size_t)(py + (i >> 2)) * e->cw + px + (i & 3)] = (uint8_t)clip1(best_pred[i] + resid[i]);
  }
  return cost;
}

static void encode_intra_mb(enc_t* e, const uint8_t* cur_nv12, int mbx, int mby, int qp) {
  mb_t* m = &e->mbs[mby * e->mbw + mbx];
  memset(m, 0, sizeof *m);
  m->type = 0;
  uint8_t cy[256], cc[2][64];
  load_cur(cur_nv12, e->cw, e->ch, mbx, mby, cy, cc);
  int has_left = avail_left(e, mbx), has_top = avail_top(e, mby);
  uint8_t* ry = plane_y(e, e->cur); uint8_t* ruv = plane_uv(e, e->cur);
  uint8_t top[16] = {0}, left[16] = {0}; int tl = 0;
  uint8_t ctop[2][8] = {{0}}, cleft[2][8] = {{0}}; int ctl[2] = {0, 0};
  if (has_top) {
    memcpy(top, ry + (size_t)(mby * 16 - 1) * e->cw + mbx * 16, 16);
    for (int x = 0; x < 8; x++) for (int c = 0; c < 2; c++) ctop[c][x] = ruv[(size_t)(mby * 8 - 1) * e->cw + (mbx * 8 + x) * 2 + c];
  }
  if (has_left) {
    for (int y = 0; y < 16; y++) left[y] = ry[(size_t)(mby * 16 + y) * e->cw + mbx * 16 - 1];
    for (int y = 0; y < 8; y++) for (int c = 0; c < 2; c++) cleft[c][y] = ruv[(size_t)(mby * 8 + y) * e->cw + (mbx * 8 - 1) * 2 + c];
  }
  if (has_top && has_left) {
    tl = ry[(size_t)(mby * 16 - 1) * e->cw + mbx * 16 - 1];
    for (int c = 0; c < 2; c++) ctl[c] = ruv[(size_t)(mby * 8 - 1) * e->cw + (mbx * 8 - 1) * 2 + c];
  }
  /* mode decisions */
  uint8_t pred[256], best_pred[256]; int best_key = 1 << 30;
  for (int mode = 0; mode < 4; mode++) {
    if ((mode == 0 && !has_top) || (mode == 1 && !has_left) || (mode == 3 && !(has_top && has_left))) continue;
    pred16(mode, top, left, tl, has_top, has_left, pred);
    int key = sad_n(cy, pred, 256) * 4 + mode;
    if (key < best_key) { best_key = key; m->i16_mode = (int8_t)mode; memcpy(best_pred, pred, 256); }
  }
  const int try_i4 = (best_key >> 2) > I4_SKIP_SAD_PER_LAMBDA * me_lambda[qp];   /* nearly flat: straight to Intra16x16 */
  uint8_t cpred[2][64], best_cpred[2][64]; best_key = 1 << 30;
  for (int mode = 0; mode < 4; mode++) {
    if ((mode == 2 && !has_top) || (mode == 1 && !has_left) || (mode == 3 && !(has_top && has_left))) continue;
    for (int c = 0; c < 2; c++) pred8c(mode, ctop[c], cleft[c], ctl[c], has_top, has_left, cpred[c]);
    int key = (sad_n(cc[0], cpred[0], 64) + sad_n(cc[1], cpred[1], 64)) * 4 + mode;
    if (key < best_key) { best_key = key; m->chroma_mode = (int8_t)mode; memcpy(best_cpred, cpred, 128); }
  }
  /* Intra4x4 candidate: run completely first (it needs its own reconstruction block by block) and saved; the
   * Intra16x16 coding below then overwrites frame and macroblock state, and the rate-distortion comparison at the
   * end restores the 4x4 result if it wins. */
  if (try_i4) intra4x4_pass(e, m, cy, mbx, mby, qp);
  mb_t m4 = *m;
  uint8_t rec4[256];
  for (int r = 0; r < 16; r++) memcpy(rec4 + 16 * r, ry + (size_t)(mby * 16 + r) * e->cw + mbx * 16, 16);
  /* luma: 16 blocks, DC separated (8.5.2) */
  int dcs[16], any_ac = 0;
  for (int b = 0; b < 16; b++) {
    int bx = blk_x[b] * 4, by = blk_y[b] * 4, res[16];
    for (int i = 0; i < 16; i++) { int p = (by + (i >> 2)) * 16 + bx + (i & 3); res[i] = cy[p] - best_pred[p]; }
    tq4x4(res, qp, 1, 1, m->coef[1 + b], &dcs[blk_y[b] * 4 + blk_x[b]]);
    int n = count_nz(m->coef[1 + b], 1, 16);
    m->nnz_l[blk_y[b] * 4 + blk_x[b]] = (uint8_t)n;
    any_ac |= n;
  }
  int hd[16], qbits = 15 + qp / 6, f = (1 << qbits) / 3;
  hadamard4x4(dcs, hd);
  int dcl[16];
  for (int k = 0; k < 16; k++) {
    int r = zigzag4x4[k];
    int v = asr(hd[r] + 1, 1);
    m->coef[0][k] = (int16_t)quant1(v, quant_mf[qp % 6][0], 2 * f, qbits + 1);
    dcl[r] = m->coef[0][k];
  }
  int fq[16], ls = 16 * dequant_v[qp % 6][0];
  hadamard4x4(dcl, fq);
  for (int b = 0; b < 16; b++) {
    int r = blk_y[b] * 4 + blk_x[b];
    int dc = qp >= 36 ? (fq[r] * ls) << (qp / 6 - 6) : asr(fq[r] * ls + (1 << (5 - qp / 6)), 6 - qp / 6);
    int resid[16];
    recon4x4(m->coef[1 + b], qp, 1, dc, resid);
    int bx = blk_x[b] * 4, by = blk_y[b] * 4;
    for (int i = 0; i < 16; i++) {
      int y = by + (i >> 2), x = bx + (i & 3);
      ry[(size_t)(mby * 16 + y) * e->cw + mbx * 16 + x] = (uint8_t)clip1(best_pred[y * 16 + x] + resid[i]);
    }
  }
  /* mode decision J = SSD + lambda_rd * bits over the luma (chroma is coded identically either way) */
  if (try_i4) {
    int64_t d16 = 0, d4 = 0;
    for (int r = 0; r < 16; r++)
      for (int c = 0; c < 16; c++) {
        int a = cy[r * 16 + c] - ry[(size_t)(mby * 16 + r) * e->cw + mbx * 16 + c], b4 = cy[r * 16 + c] - rec4[r * 16 + c];
        d16 += a * a; d4 += b4 * b4;
      }
    bitw_t b; bw_init(&b);
    cavlc_block(&b, m->coef[0], 0, 16, -2);
    if (any_ac) for (int blk = 0; blk < 16; blk++) cavlc_block(&b, m->coef[1 + blk], 1, 15, -2);
    int bits16 = 8 + (int)bw_bits(&b);
    bw_free(&b); bw_init(&b);
    int cbp4 = 0, bits4 = 8;
    for (int blk = 0; blk < 16; blk++) if (m4.nnz_l[blk_y[blk] * 4 + blk_x[blk]]) cbp4 |= 1 << (blk >> 2);
    for (int blk = 0; blk < 16; blk++) {
      if (cbp4 & (1 << (blk >> 2))) cavlc_block(&b, m4.coef[1 + blk], 0, 16, -2);
      /* the mode bits are recomputed against the I4 state, which is what the entropy coder will see */
    }
    bits4 += (int)bw_bits(&b);
    bw_free(&b);
    { mb_t keep = *m; *m = m4;      /* i4_pred_mode() reads the macroblock's own modes */
      for (int blk = 0; blk < 16; blk++) bits4 += m4.i4_modes[blk_y[blk] * 4 + blk_x[blk]] == i4_pred_mode(e, mbx, mby, blk_x[blk], blk_y[blk]) ? 1 : 4;
      *m = keep; }
    const int64_t l2 = rd_lambda[qp];
    if (d4 + l2 * bits4 < d16 + l2 * bits16 && !e->no_i4) {
      int8_t cm = m->chroma_mode;
      *m = m4; m->type = 3; m->chroma_mode = cm;
      for (int r = 0; r < 16; r++) memcpy(ry + (size_t)(mby * 16 + r) * e->cw + mbx * 16, rec4 + 16 * r, 16);
      any_ac = 0;
      int cbp_c4 = code_chroma(e, m, mbx, mby, qp, 1, cc, best_cpred);
      m->cbp = (uint8_t)(cbp4 | (cbp_c4 << 4));
      make_pcm_if_too_big(e, m, cur_nv12, mbx, mby);
      return;
    }
  }
  int cbp_c = code_chroma(e, m, mbx, mby, qp, 1, cc, best_cpred);
  m->cbp = (uint8_t)((any_ac ? 15 : 0) | (cbp_c << 4));
  make_pcm_if_too_big(e, m, cur_nv12, mbx, mby);
}

/* ------------------------------------------------------------------ inter macroblock (8.4) */
#define ME_EARLY_SAD_PER_LAMBDA 96
#define ME_REFINE_MAX_SAD 8192             /* no sub-sample refinement of a full-sample match this bad (DESIGN.md 5.3) */
#define ME_NEWCONTENT_DY 2                 /* vertical range of the reduced search on new content (DESIGN.md 5.3) */
#define ME_PRED_SAD_FACTOR 4
#define ME_FRAC_PENALTY_BITS 4   /* fractional vectors pay 4 extra bits: they cost more mvd bits than the zero-relative estimate sees */
static int se_bits(int v) { unsigned c = v > 0 ? 2u * v - 1 : (unsigned)(-2 * v); int len = 0; c += 1; while ((c >> len) > 1) len++; return 2 * len + 1; }

/* 8.4.2.2.1: predicted 16x16 luma block for a quarter-sample offset (qx,qy) in [-3,3] from the full-sample position the
 * planes were built around.  Every fractional position is one plane or the rounded average of two (Table 8-12):
 *   G integer, b horizontal half, h vertical half, j centre; a,c,d,n,e,f,g,i,k,p,q,r = averages. */
static void luma_mc_planes(uint8_t Gp[22][22], uint8_t bq[18][17], uint8_t hq[17][18], uint8_t jq[17][17], int qx, int qy, uint8_t out[256]) {
  const int xi = asr(qx, 2), yi = asr(qy, 2), fx = qx & 3, fy = qy & 3;
  for (int y = 0; y < 16; y++)
    for (int x = 0; x < 16; x++) {
      const int X = x + xi, Y = y + yi;
      const int G = Gp[Y + 3][X + 3], H = Gp[Y + 3][X + 4], M = Gp[Y + 4][X + 3];
      const int b = bq[Y + 1][X + 1], s = bq[Y + 2][X + 1], h = hq[Y + 1][X + 1], mm = hq[Y + 1][X + 2], j = jq[Y + 1][X + 1];
      int v;
      switch (fy * 4 + fx) {
        case 0: v = G; break;
        case 1: v = (G + b + 1) >> 1; break;
        case 2: v = b; break;
        case 3: v = (H + b + 1) >> 1; break;
        case 4: v = (G + h + 1) >> 1; break;
        case 5: v = (b + h + 1) >> 1; break;
        case 6: v = (b + j + 1) >> 1; break;
        case 7: v = (b + mm + 1) >> 1; break;
        case 8: v = h; break;
        case 9: v = (h + j + 1) >> 1; break;
        case 10: v = j; break;
        case 11: v = (j + mm + 1) >> 1; break;
        case 12: v = (M + h + 1) >> 1; break;
        case 13: v = (h + s + 1) >> 1; break;
        case 14: v = (j + s + 1) >> 1; break;
        default: v = (mm + s + 1) >> 1; break;
      }
      out[y * 16 + x] = (uint8_t)v;
    }
}

/* macroblock rows [r0, r1) of the band (stripe) holding row mby; the whole picture when striping is off */
static void band_rows(const enc_t* e, int mby, int* r0, int* r1) {
  if (!e->stripe_rows) { *r0 = 0; *r1 = e->mbh; return; }
  *r0 = mby / e->stripe_rows * e->stripe_rows;
  *r1 = *r0 + e->stripe_rows; if (*r1 > e->mbh) *r1 = e->mbh;
}

/* Anchor macroblocks: one per 4x4 group of macroblocks (rows counted from the band's first row), at offset (1,1) of its group
 * (clamped into the band / picture).  The anchors of a P picture are analysed first; when the temporal predictor of any other
 * macroblock fails, the vector its group's anchor has just found is tried before the exhaustive search — coherent motion that
 * STARTS in this picture (a scroll or pan after a still or a cut, where last picture's vectors are useless) is then searched for
 * once per sixteen macroblocks instead of once per macroblock. */
static void anchor_of(const enc_t* e, int mbx, int mby, int* ax, int* ay) {
  int br0, br1; band_rows(e, mby, &br0, &br1);
  *ax = 4 * (mbx / 4) + 1; if (*ax > e->mbw - 1) *ax = e->mbw - 1;
  *ay = br0 + 4 * ((mby - br0) / 4) + 1; if (*ay > br1 - 1) *ay = br1 - 1;
}
static int is_anchor(const enc_t* e, int mbx, int mby) { int ax, ay; anchor_of(e, mbx, mby, &ax, &ay); return ax == mbx && ay == mby; }

/* candidate (cdx,cdy), full-sample — the zero vector included: "this macroblock did not move last picture" is a prediction too, and
 * static content whose co-located SAD sits just above the early-termination threshold (noise, text at a coarse QP) would otherwise
 * run the exhaustive search only to find (0,0) again.  Accepted when its SAD is within 4x the noise threshold AND it is a strict
 * local minimum of the cost over its 8 full-sample neighbours AND it costs no more than the zero vector; *key = its search key */
static int try_candidate(const uint8_t cy[256], uint8_t win[48][48], int cdx, int cdy, int lambda, int sad0, uint32_t* key) {
  if (cdx < -15 || cdx > 14 || cdy < -15 || cdy > 15) return 0;
  uint32_t kc = 0, kmin = 0xffffffffu;
  for (int j = -1; j <= 1; j++)
    for (int i = -1; i <= 1; i++) {
      int sad = 0;
      for (int r = 0; r < 16; r++) for (int c = 0; c < 16; c++) sad += iabs(cy[r * 16 + c] - win[16 + cdy + j + r][16 + cdx + i + c]);
      const uint32_t cost = (uint32_t)(sad + lambda * (se_bits(4 * (cdx + i)) + se_bits(4 * (cdy + j))));
      const uint32_t k = (cost << 11) | (uint32_t)((cdy + j + 16) * 32 + (cdx + i + 16));
      if (i == 0 && j == 0) kc = k; else if (k < kmin) kmin = k;
    }
  const int sadc = (int)(kc >> 11) - lambda * (se_bits(4 * cdx) + se_bits(4 * cdy));
  const uint32_t key0 = ((uint32_t)(sad0 + 2 * lambda) << 11) | (16 * 32 + 16);     /* the zero vector's own key */
  if (sadc <= ME_PRED_SAD_FACTOR * ME_EARLY_SAD_PER_LAMBDA * lambda && kc < kmin && kc <= key0) { *key = kc; return 1; }
  return 0;
}

static void encode_inter_mb(enc_t* e, const uint8_t* cur_nv12, int mbx, int mby, int qp) {
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
  if (search && prev_type == 1 && !e->no_tpred) {
    const int cdx = asr(prev_mvx + 2, 2), cdy = asr(prev_mvy + 2, 2);
    tried_zero = !(cdx | cdy);
    if ((!tried_zero || !e->no_zcand) && try_candidate(cy, win, cdx, cdy, lambda, sad0, &best)) { search = 0; pred_hit = 1; bdx = cdx; bdy = cdy; src_mvx = prev_mvx; src_mvy = prev_mvy; }
  }
  /* anchor predictor: the vector the anchor of this macroblock's 4x4 group found in THIS picture (anchors run first) */
  if (search && !e->no_tpred && !e->no_anchor && !is_anchor(e, mbx, mby)) {
    int ax, ay; anchor_of(e, mbx, mby, &ax, &ay);
    const mb_t* a = &e->mbs[ay * e->mbw + ax];
    const int cdx = asr(a->me_mv[0] + 2, 2), cdy = asr(a->me_mv[1] + 2, 2);
    const int skip_zero = !(cdx | cdy) && (tried_zero || e->no_zcand);      /* the zero vector is not tested twice */
    if (!skip_zero && try_candidate(cy, win, cdx, cdy, lambda, sad0, &best)) { search = 0; pred_hit = 1; bdx = cdx; bdy = cdy; src_mvx = a->me_mv[0]; src_mvy = a->me_mv[1]; }
    /* new content: the anchor's exhaustive search found no match worth the name and this macroblock's co-located block is as far
     * off — another 1089-candidate search would only pick the least bad of the noise.  The search shrinks to the five rows
     * around dy = 0 (160 candidates: most of what picking a minimum among noise buys, for a sixth of the work). */
    else if (a->me_bad && sad0 >= ME_REFINE_MAX_SAD && !e->no_newcontent) dyr = ME_NEWCONTENT_DY;
  }
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
  /* ---- quarter-sample refinement (8.4.2.2.1).  Around the best full-sample position (only when its 6-tap support
   * [-3,+18] lies inside the 48x48 window, i.e. |dx|,|dy| <= 13, and the search ran): the half-sample planes
   *   b1 = E - 5F + 20G + 20H - 5I + J (unrounded), b = clip((b1+16)>>5), h likewise vertically, j = clip((6-tap of b1 + 512)>>10)
   * are built once; stage H tries the 8 half-sample neighbours, stage Q the 8 quarter-sample neighbours of the stage-H
   * winner; cost = SAD + lambda*(bits(mvx)+bits(mvy) + 4 if fractional), key = cost<<4 | candidate index (0 = centre wins ties). */
  int mvx = 4 * bdx, mvy = 4 * bdy;
  uint8_t py[256], pc[2][64];
  int have_planes = 0;
  static const int8_t nb8[8][2] = { {-1,-1}, {0,-1}, {1,-1}, {-1,0}, {1,0}, {-1,1}, {0,1}, {1,1} };
  uint8_t Gp[22][22], bq[18][17], hq[17][18], jq[17][17];   /* Gp[v+3][u+3], bq[v+1][u+1], hq[v+1][u+1], jq[v+1][u+1] */
  /* not worth refining when the full-sample match is already within the quantisation noise of this QP */
  const int sad_int = (int)(best >> 11) - lambda * (se_bits(4 * bdx) + se_bits(4 * bdy));
  m->me_bad = (search || pred_hit) && sad_int >= ME_REFINE_MAX_SAD;     /* however the vector was found: nothing here matches */
  /* a predictor hit whose previous vector was full-sample is not refined again: the previous refinement already preferred it */
  const int pred_frac = pred_hit && ((src_mvx | src_mvy) & 3);
  /* ... nor when it is hopeless (mean absolute difference of 32 per sample and more: new content, nothing to polish) */
  if ((search || pred_frac) && iabs(bdx) <= 13 && iabs(bdy) <= 13 && sad_int > ME_EARLY_SAD_PER_LAMBDA * lambda && (e->no_refine_cap || sad_int < ME_REFINE_MAX_SAD)) {
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
        const uint32_t cost = (uint32_t)(sad_n(cy, pr, 256) + lambda * (se_bits(4 * bdx + qx) + se_bits(4 * bdy + qy) + (((qx | qy) & 3) ? ME_FRAC_PENALTY_BITS : 0)));
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
      for (int c = 0; c < 16; c++) py[r * 16 + c] = refy[(size_t)clip3(ylo, yhi, y0 + bdy + r) * e->cw + clip3(0, e->cw - 1, x0 + bdx + c)];
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
  make_pcm_if_too_big(e, m, cur_nv12, mbx, mby);
}

/* ------------------------------------------------------------------ CAVLC (9.2) */
static void cavlc_block(bitw_t* b, const int16_t* lv, int start, int maxc, int nC) {
  /* lv[start .. start+maxc) in scan order */
  int idx[16], n = 0;
  for (int k = 0; k < maxc; k++) if (lv[start + k]) idx[n++] = k;
  int total = n, t1 = 0;
  for (int i = n - 1; i >= 0 && t1 < 3; i--) { if (iabs(lv[start + idx[i]]) == 1) t1++; else break; }
  if (nC == -1) bw_put(b, chroma_dc_coeff_token_len[4 * total + t1], chroma_dc_coeff_token_bits[4 * total + t1]);
  else if (nC == -2) {   /* size estimate before the neighbours are known: the longest coeff_token of the four tables */
    int len = 0;
    for (int t = 0; t < 4; t++) if (coeff_token_len[t][4 * total + t1] > len) len = coeff_token_len[t][4 * total + t1];
    bw_put(b, len, 0);
  } else {
    int tab = nC < 2 ? 0 : nC < 4 ? 1 : nC < 8 ? 2 : 3;
    bw_put(b, coeff_token_len[tab][4 * total + t1], coeff_token_bits[tab][4 * total + t1]);
  }
  if (!total) return;
  for (int i = 0; i < t1; i++) bw_put(b, 1, lv[start + idx[n - 1 - i]] < 0);
  int suffix_len = (total > 10 && t1 < 3) ? 1 : 0;
  for (int i = t1; i < total; i++) {
    int level = lv[start + idx[n - 1 - i]];
    int code = level > 0 ? 2 * level - 2 : -2 * level - 1;
    if (i == t1 && t1 < 3) code -= 2;
    if (suffix_len == 0) {
      if (code < 14) { bw_put(b, code, 0); bw_put(b, 1, 1); }
      else if (code < 30) { bw_put(b, 14, 0); bw_put(b, 1, 1); bw_put(b, 4, code - 14); }
      else { bw_put(b, 15, 0); bw_put(b, 1, 1); bw_put(b, 12, code - 30); }
    } else {
      if (code < (15 << suffix_len)) { bw_put(b, code >> suffix_len, 0); bw_put(b, 1, 1); bw_put(b, suffix_len, code & ((1 << suffix_len) - 1)); }
      else { bw_put(b, 15, 0); bw_put(b, 1, 1); bw_put(b, 12, code - (15 << suffix_len)); }
    }
    if (suffix_len == 0) suffix_len = 1;
    if (iabs(level) > (3 << (suffix_len - 1)) && suffix_len < 6) suffix_len++;
  }
  int zeros = idx[n - 1] + 1 - total;          /* total_zeros */
  if (total < maxc) {
    if (nC == -1) bw_put(b, chroma_dc_total_zeros_len[total - 1][zeros], chroma_dc_total_zeros_bits[total - 1][zeros]);
    else bw_put(b, total_zeros_len[total - 1][zeros], total_zeros_bits[total - 1][zeros]);
  }
  int left = zeros;
  for (int i = n - 1; i > 0 && left > 0; i--) {
    int run = idx[i] - idx[i - 1] - 1;
    int t = (left > 7 ? 7 : left) - 1;
    bw_put(b, run_len[t][run], run_bits[t][run]);
    left -= run;
  }
}

/* nC for luma block (bx,by in 4-sample units) / chroma block: 9.2.1 */
static int mb_avail(const enc_t* e, int mbx, int mby, int nx, int ny) {
  if (nx < 0 || nx >= e->mbw || ny < 0) return 0;
  if (ny != mby && !avail_top(e, mby)) return 0;
  if (nx != mbx && !avail_left(e, mbx)) return 0;
  return 1;
}
static int nnz_luma_at(const enc_t* e, const uint8_t* skip, int mbx, int mby, int bx, int by, int* ok) {
  int nx = mbx, ny = mby;
  if (bx < 0) { nx--; bx += 4; }
  if (by < 0) { ny--; by += 4; }
  *ok = mb_avail(e, mbx, mby, nx, ny);
  if (!*ok) return 0;
  const mb_t* n = &e->mbs[ny * e->mbw + nx];
  if (skip[ny * e->mbw + nx]) return 0;
  if (n->type == 2) return 16;
  return n->nnz_l[by * 4 + bx];
}
static int nnz_chroma_at(const enc_t* e, const uint8_t* skip, int mbx, int mby, int c, int bx, int by, int* ok) {
  int nx = mbx, ny = mby;
  if (bx < 0) { nx--; bx += 2; }
  if (by < 0) { ny--; by += 2; }
  *ok = mb_avail(e, mbx, mby, nx, ny);
  if (!*ok) return 0;
  const mb_t* n = &e->mbs[ny * e->mbw + nx];
  if (skip[ny * e->mbw + nx]) return 0;
  if (n->type == 2) return 16;
  return n->nnz_c[c][by * 2 + bx];
}
static int calc_nc(int na, int oka, int nb, int okb) { return oka && okb ? (na + nb + 1) >> 1 : oka ? na : okb ? nb : 0; }

/* motion vector prediction for a 16x16 partition (8.4.1.3) and the P_Skip inference (8.4.1.1).
 * Inter macroblocks have refIdx 0; intra (here: I_PCM) and unavailable neighbours count as refIdx -1, mv 0. */
static void mv_neighbours(const enc_t* e, int mbx, int mby, int av[3], int ref0[3], int mv[3][2]) {
  int top = avail_top(e, mby);
  int nx[3] = { mbx - 1, mbx, mbx + 1 }, ny[3] = { mby, mby - 1, mby - 1 };
  av[0] = avail_left(e, mbx); av[1] = top; av[2] = top && mbx + 1 < e->mbw;
  if (!av[2]) { nx[2] = mbx - 1; av[2] = top && mbx > 0; }    /* C unavailable -> D */
  for (int i = 0; i < 3; i++) {
    mv[i][0] = mv[i][1] = 0; ref0[i] = 0;
    if (av[i]) {
      const mb_t* n = &e->mbs[ny[i] * e->mbw + nx[i]];
      if (n->type == 1) { ref0[i] = 1; mv[i][0] = n->mv[0]; mv[i][1] = n->mv[1]; }
    }
  }
}
static int median3(int a, int b, int c) { int mx = a > b ? a : b, mn = a < b ? a : b; return c > mx ? mx : (c < mn ? mn : c); }
static void mv_pred16(const enc_t* e, int mbx, int mby, int out[2]) {
  int av[3], r0[3], mv[3][2];
  mv_neighbours(e, mbx, mby, av, r0, mv);
  if (!av[1] && !av[2] && av[0]) { out[0] = mv[0][0]; out[1] = mv[0][1]; return; }   /* B, C unavailable: all three become A */
  int cnt = r0[0] + r0[1] + r0[2];
  if (cnt == 1) { int i = r0[0] ? 0 : r0[1] ? 1 : 2; out[0] = mv[i][0]; out[1] = mv[i][1]; return; }
  out[0] = median3(mv[0][0], mv[1][0], mv[2][0]);
  out[1] = median3(mv[0][1], mv[1][1], mv[2][1]);
}
static void mv_pred_skip(const enc_t* e, int mbx, int mby, int out[2]) {
  int okA = avail_left(e, mbx), okB = avail_top(e, mby);
  out[0] = out[1] = 0;
  if (!okA || !okB) return;
  const mb_t* a = &e->mbs[mby * e->mbw + mbx - 1]; const mb_t* b = &e->mbs[(mby - 1) * e->mbw + mbx];
  if ((a->type == 1 && a->mv[0] == 0 && a->mv[1] == 0) || (b->type == 1 && b->mv[0] == 0 && b->mv[1] == 0)) return;
  mv_pred16(e, mbx, mby, out);
}

/* Upper bound of the macroblock_layer() size: exact CAVLC cost of every coded block with the longest
 * coeff_token of the four nC tables, plus 48 bits for mb_type / mvd / cbp / qp_delta.  A macroblock whose bound
 * exceeds the 3200-bit limit of A.3.1 is sent as I_PCM instead (decided at analysis time because the
 * reconstruction — which the following macroblocks predict from — becomes the source samples). */
#define MB_BITS_LIMIT 3200
static int mb_bits_estimate(const mb_t* m) {
  bitw_t b; bw_init(&b);
  if (m->type == 0) cavlc_block(&b, m->coef[0], 0, 16, -2);
  if (m->type == 3) bw_put(&b, 32, 0), bw_put(&b, 16, 0);   /* Intra4x4: up to 64 bits of prediction modes -> 96-bit header budget */
  for (int blk = 0; blk < 16; blk++) {
    if (!(m->cbp & (1 << (blk >> 2)))) continue;
    if (m->type == 0) cavlc_block(&b, m->coef[1 + blk], 1, 15, -2); else cavlc_block(&b, m->coef[1 + blk], 0, 16, -2);
  }
  int cc = m->cbp >> 4;
  if (cc) { cavlc_block(&b, m->coef[17], 0, 4, -1); cavlc_block(&b, m->coef[18], 0, 4, -1); }
  if (cc & 2) for (int k = 0; k < 8; k++) cavlc_block(&b, m->coef[19 + k], 1, 15, -2);
  int bits = 48 + (int)bw_bits(&b);
  bw_free(&b);
  return bits;
}
static void make_pcm_if_too_big(enc_t* e, mb_t* m, const uint8_t* cur_nv12, int mbx, int mby) {
  if (mb_bits_estimate(m) <= MB_BITS_LIMIT) return;
  uint8_t* ry = plane_y(e, e->cur); uint8_t* ruv = plane_uv(e, e->cur);
  const uint8_t* cuv = cur_nv12 + (size_t)e->cw * e->ch;
  for (int r = 0; r < 16; r++) memcpy(ry + (size_t)(mby * 16 + r) * e->cw + mbx * 16, cur_nv12 + (size_t)(mby * 16 + r) * e->cw + mbx * 16, 16);
  for (int r = 0; r < 8; r++) memcpy(ruv + (size_t)(mby * 8 + r) * e->cw + mbx * 16, cuv + (size_t)(mby * 8 + r) * e->cw + mbx * 16, 16);
  m->type = 2; m->cbp = 0; m->mv[0] = m->mv[1] = 0;
  memset(m->nnz_l, 16, sizeof m->nnz_l); memset(m->nnz_c, 16, sizeof m->nnz_c);
}

static void write_residual(const enc_t* e, bitw_t* b, const uint8_t* skip, const mb_t* m, int mbx, int mby) {
  int oka, okb, na, nb;
  if (m->type == 0) {   /* Intra16x16DCLevel: nC as for luma block 0 */
    na = nnz_luma_at(e, skip, mbx, mby, -1, 0, &oka); nb = nnz_luma_at(e, skip, mbx, mby, 0, -1, &okb);
    cavlc_block(b, m->coef[0], 0, 16, calc_nc(na, oka, nb, okb));
  }
  for (int blk = 0; blk < 16; blk++) {
    if (!(m->cbp & (1 << (blk >> 2)))) continue;
    int bx = blk_x[blk], by = blk_y[blk];
    na = nnz_luma_at(e, skip, mbx, mby, bx - 1, by, &oka); nb = nnz_luma_at(e, skip, mbx, mby, bx, by - 1, &okb);
    if (m->type == 0) cavlc_block(b, m->coef[1 + blk], 1, 15, calc_nc(na, oka, nb, okb));
    else cavlc_block(b, m->coef[1 + blk], 0, 16, calc_nc(na, oka, nb, okb));
  }
  int cc = m->cbp >> 4;
  if (cc) { cavlc_block(b, m->coef[17], 0, 4, -1); cavlc_block(b, m->coef[18], 0, 4, -1); }
  if (cc & 2)
    for (int c = 0; c < 2; c++)
      for (int blk = 0; blk < 4; blk++) {
        int bx = blk & 1, by = blk >> 1;
        na = nnz_chroma_at(e, skip, mbx, mby, c, bx - 1, by, &oka); nb = nnz_chroma_at(e, skip, mbx, mby, c, bx, by - 1, &okb);
        cavlc_block(b, m->coef[19 + c * 4 + blk], 1, 15, calc_nc(na, oka, nb, okb));
      }
}

/* 7.3.3 slice header */
static void write_slice_header(const enc_t* e, bitw_t* b, int first_mb, int idr, int qp, int frame_num) {
  bw_ue(b, first_mb);
  bw_ue(b, idr ? 7 : 5);                       /* slice_type: all slices of the picture I / P */
  bw_ue(b, 0);                                 /* pic_parameter_set_id */
  bw_put(b, 8, frame_num & 255);
  if (idr) bw_ue(b, e->idr_count & 15);        /* idr_pic_id */
  if (!idr) { bw_put(b, 1, 0); bw_put(b, 1, 0); }   /* num_ref_idx_active_override_flag, ref_pic_list_modification_flag_l0 */
  if (idr) { bw_put(b, 1, 0); bw_put(b, 1, 0); }    /* no_output_of_prior_pics_flag, long_term_reference_flag */
  else bw_put(b, 1, 0);                             /* adaptive_ref_pic_marking_mode_flag */
  bw_se(b, qp - 26);                           /* slice_qp_delta */
  bw_ue(b, 1);                                 /* disable_deblocking_filter_idc */
}

/* entropy-code one slice (7.3.4, 7.3.5) into a NAL appended at out; returns bytes written */
static size_t code_slice(enc_t* e, int s, int idr, int qp, uint8_t* skip, uint8_t* out, int64_t* bits) {
  bitw_t b; bw_init(&b);
  int row0 = s * e->slice_rows, row1 = row0 + e->slice_rows, x0 = 0, x1 = e->mbw;
  if (e->pic_seg) { const int segs = pic_segs(e); row0 = s / segs; row1 = row0 + 1; x0 = (s % segs) * e->pic_seg; x1 = x0 + e->pic_seg; if (x1 > e->mbw) x1 = e->mbw; }
  if (row1 > e->mbh) row1 = e->mbh;
  int br0, br1; band_rows(e, row0, &br0, &br1);
  const int first_nal_of_au = row0 == br0 && x0 == 0 && !idr;     /* 4-byte start code opens each band's access unit */
  write_slice_header(e, &b, (row0 - br0) * e->mbw + x0, idr, qp, idr ? 0 : e->stripe_rows ? e->stripe_fn[row0 / e->stripe_rows] : e->frame_num);
  int skip_run = 0;
  for (int mby = row0; mby < row1; mby++)
    for (int mbx = x0; mbx < x1; mbx++) {
      const mb_t* m = &e->mbs[mby * e->mbw + mbx];
      if (!idr) {
        int sp[2];
        mv_pred_skip(e, mbx, mby, sp);
        if (m->type == 1 && m->cbp == 0 && m->mv[0] == sp[0] && m->mv[1] == sp[1]) { skip[mby * e->mbw + mbx] = 1; skip_run++; continue; }
        bw_ue(&b, skip_run); skip_run = 0;
      }
      if (m->type == 2) {                       /* I_PCM (7.3.5): mb_type 25 (+5 in P slices), alignment, raw samples */
        bw_ue(&b, idr ? 25 : 30);
        if (b.nacc) bw_put(&b, 8 - b.nacc, 0);  /* pcm_alignment_zero_bit */
        const uint8_t* ry = plane_y(e, e->cur); const uint8_t* ruv = plane_uv(e, e->cur);
        for (int r = 0; r < 16; r++) for (int c = 0; c < 16; c++) bw_put(&b, 8, ry[(size_t)(mby * 16 + r) * e->cw + mbx * 16 + c]);
        for (int k = 0; k < 2; k++)
          for (int r = 0; r < 8; r++) for (int c = 0; c < 8; c++) bw_put(&b, 8, ruv[(size_t)(mby * 8 + r) * e->cw + (mbx * 8 + c) * 2 + k]);
        continue;
      }
      if (m->type == 3) {                       /* I_NxN with Intra4x4 (7.3.5, 7.3.5.1) */
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
        bw_se(&b, 0);                          /* mb_qp_delta */
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
  size_t n = nal_write(out, first_nal_of_au, idr ? 3 : 2, idr ? 5 : 1, b.buf, b.pos);
  bw_free(&b);
  return n;
}

/* ------------------------------------------------------------------ rate control (DESIGN.md §5.6) */
static int rc_initial_qp(int64_t target_bits, int mbs) {
  int64_t per_mb = target_bits / (mbs > 0 ? mbs : 1);
  return per_mb >= 400 ? 22 : per_mb >= 200 ? 26 : per_mb >= 100 ? 30 : per_mb >= 50 ? 34 : per_mb >= 25 ? 38 : 42;
}
/* Quantiser step in Q6 (64 * 2^(qp/6)): the P-picture model is  bits(qp) = X / QS[qp]. */
#define RC_DEBT_PICTURES 32
static const int32_t RC_QS[52] = {
  64, 72, 81, 91, 102, 114, 128, 144, 161, 181, 203, 228, 256, 287, 323, 362, 406, 456, 512, 575, 645, 724, 813, 912, 1024, 1149,
  1290, 1448, 1625, 1825, 2048, 2299, 2580, 2896, 3251, 3649, 4096, 4598, 5161, 5793, 6502, 7298, 8192, 9195, 10321, 11585, 13004,
  14596, 16384, 18390, 20643, 23170 };
#define RC_QP_MIN 10
#define RC_QP_MAX 51
#define RC_STATIC_PARK (1 << 20)

/* QP of picture k from the feedback record it may see (the state after picture k-2). */
static int rc_frame_qp(const enc_t* e, const struct rcfb* fb, int idr, int rc_mode, int qp_fixed, int64_t target_bits) {
  const int mbs = e->mbw * e->mbh;
  const int paint = e->paint_trigger > 0 && !idr && fb->paint;
  if (rc_mode == 1) return clip3(0, 51, paint ? e->paint_qp : qp_fixed);
  int q = fb->qp < 0 ? rc_initial_qp(target_bits, mbs) : fb->qp;
  /* an IDR requested in mid-stream (PLI, resize) is not coded finer than a fresh start with 4x the picture budget would be */
  if (idr) { int q0 = rc_initial_qp(4 * target_bits, mbs); if (q < q0) q = q0; }
  if (paint && e->paint_qp < q) q = clip3(0, 51, e->paint_qp);
  return q;
}

/* After picture k (its RBSP bit count is known): advance the feedback record.  prev = the record after picture k-1,
 * used = the record picture k was coded from (after k-2).  Deterministic integer arithmetic: the GPU runs the same code. */
static void rc_step(const enc_t* e, struct rcfb* out, const struct rcfb* prev, const struct rcfb* used, int64_t bits, int qp_used,
                    int idr, int coded, int rc_mode, int64_t target) {
  struct rcfb n = *prev;
  n.debt = 0;
  const int was_paint = e->paint_trigger > 0 && !idr && used->paint;
  /* paint-over scheduler: count all-skipped pictures; at `paint_trigger` schedule `paint_burst` pictures at the paint-over QP
   * (each step schedules the picture two ahead); real motion cancels what is left of the burst */
  if (idr || (coded && !was_paint)) { n.static_run = 0; n.remaining = 0; }
  else if (!coded) {
    n.static_run = prev->static_run + 1 > RC_STATIC_PARK ? RC_STATIC_PARK : prev->static_run + 1;
    if (e->paint_trigger > 0 && n.static_run == e->paint_trigger) n.remaining = e->paint_burst > 0 ? e->paint_burst : 1;
  }
  n.paint = n.remaining > 0;
  if (n.paint) n.remaining--;
  if (rc_mode == 0) {
    const int64_t T = target < 1 ? 1 : target;
    const int mbs = e->mbw * e->mbh;
    int64_t full = prev->fullness + bits - T;
    if (full < -4 * T) full = -4 * T;         /* at most four pictures' worth of unspent budget is carried forward */
    if (full > 64 * T) full = 64 * T;
    n.fullness = full;
    int64_t budget = T - full / 16;            /* repay (or spend) the bucket over about 16 pictures */
    if (budget < T / 2) budget = T / 2;
    if (budget > 2 * T) budget = 2 * T;
    const int base = prev->qp < 0 ? rc_initial_qp(T, mbs) : prev->qp;     /* the decision already in flight (for picture k+1) */
    int q = base;
    /* X = this picture's complexity, bits x quantiser step (key frames: 0 = unknown).  Decisions compare the last TWO pictures:
     * a single large picture (a refinement after a QP decrease, a scroll restart) is paid for through the bucket, only a
     * SUSTAINED overshoot makes the quantiser coarser; and they are absolute (relative to the QP the picture was coded with),
     * so the two-picture feedback delay does not make the controller react twice to the same overshoot. */
    n.X = idr ? 0 : bits * RC_QS[qp_used];
    if (!idr) {
      const int64_t lim = budget * RC_QS[qp_used];
      const int64_t lo = prev->X > 0 && prev->X < n.X ? prev->X : n.X, hi = prev->X > n.X ? prev->X : n.X;
      /* the level the overshoot is judged on: the smaller of the two pictures when one towers over the other (a spike),
       * their mean otherwise (alternating sizes) */
      const int64_t eff = hi > 3 * lo ? lo : (lo + hi) / 2;
      int qt = base;
      if (eff * 100 > lim * 104) {
        static const int thr[9] = {104, 119, 133, 150, 168, 189, 238, 300, 378}, stp[9] = {1, 2, 3, 4, 5, 6, 8, 10, 12};
        int dq = 1;
        for (int i = 0; i < 9; i++) if (eff * 100 > lim * thr[i]) dq = stp[i];
        qt = qp_used + dq;
      } else if (hi * 100 < lim * 88 && full <= 0) {
        qt = qp_used - ((hi * 2 < lim && full < -2 * T) ? 2 : 1);
      }
      /* debt: spikes the two-picture rule lets through (a scroll that restarts every N pictures, recurring cuts) pile up in the
       * bucket; while it holds more than RC_DEBT_PICTURES pictures' worth, a picture that coded anything makes the quantiser one
       * step coarser whatever the last two pictures say — and (rule above) it gets finer again only once the bucket is empty */
      if (full > RC_DEBT_PICTURES * T && coded && qt <= qp_used) { qt = qp_used + 1; n.debt = 1; }
      q = clip3(base - 2, base + 4, qt);
    }
    n.qp = clip3(RC_QP_MIN, RC_QP_MAX, q);
  }
  *out = n;
}

/* ------------------------------------------------------------------ public API */
void* b2v_ref_enc_create(int width, int height, int slice_rows) {
  enc_t* e = (enc_t*)calloc(1, sizeof *e);
  e->width = width; e->height = height;
  e->cw = (width + 15) & ~15; e->ch = (height + 15) & ~15;
  e->mbw = e->cw / 16; e->mbh = e->ch / 16;
  /* slice_rows <= 0: the default rule — P pictures in slices of 8 macroblock rows (one slice per band in striped mode).  Inside a slice
   * a macroblock sees the row above: its motion vector is predicted from there and P_Skip infers a moving vector, so a scrolling
   * region costs no bits per macroblock; with one row per slice every moving macroblock pays ~7 bits of header (4K scrolling text at
   * QP 33: 30.2 KB per P picture with 1 row, 22.3 / 18.0 / 15.8 KB with 2 / 4 / 8 rows, 13.7 KB with one slice per picture).
   * IDR pictures have their own, finer slicing (seg_cols below) whatever slice_rows is. */
  e->auto_rows = slice_rows <= 0;
  e->slice_rows = slice_rows > 0 ? slice_rows : (e->mbh < DEFAULT_SLICE_ROWS ? e->mbh : DEFAULT_SLICE_ROWS);
  e->n_slices = (e->mbh + e->slice_rows - 1) / e->slice_rows;
  size_t fb = (size_t)e->cw * e->ch * 3 / 2;
  e->recon[0] = (uint8_t*)calloc(fb, 1); e->recon[1] = (uint8_t*)calloc(fb, 1);
  e->mbs = (mb_t*)calloc((size_t)e->mbw * e->mbh, sizeof(mb_t));
  e->fb[0].qp = e->fb[1].qp = -1; e->paint_burst = 1;
  e->seg_cols = auto_seg_cols(e->mbw, e->mbh);
  e->no_i4 = getenv("B2V_REF_NO_I4") != NULL; e->no_tpred = getenv("B2V_REF_NO_TPRED") != NULL; e->no_refine_cap = getenv("B2V_REF_NO_REFINE_CAP") != NULL; e->no_anchor = getenv("B2V_REF_NO_ANCHOR") != NULL; e->no_newcontent = getenv("B2V_REF_NO_NEWCONTENT") != NULL; e->no_zcand = getenv("B2V_REF_NO_ZCAND") != NULL;
  write_param_sets(e);
  return e;
}
void b2v_ref_enc_destroy(void* h) {
  enc_t* e = (enc_t*)h;
  if (!e) return;
  free(e->recon[0]); free(e->recon[1]); free(e->mbs); free(e);
}
int b2v_ref_enc_coded_w(void* h) { return ((enc_t*)h)->cw; }
int b2v_ref_enc_coded_h(void* h) { return ((enc_t*)h)->ch; }
const uint8_t* b2v_ref_enc_recon(void* h) { enc_t* e = (enc_t*)h; return e->recon[e->cur]; }
int b2v_ref_enc_last_qp(void* h) { return ((enc_t*)h)->last_qp; }
/* the feedback record written after the last picture (test hook: which rate-control and paint-over branches a stream reaches):
 * out = {fullness, qp, static_run, remaining, paint, debt}; returns 0, or -1 before the first picture */
int b2v_ref_enc_rc_state(void* h, int64_t* out) {
  enc_t* e = (enc_t*)h;
  if (e->pic == 0) return -1;
  const struct rcfb* r = &e->fb[(e->pic - 1) & 1];
  out[0] = r->fullness; out[1] = r->qp; out[2] = r->static_run; out[3] = r->remaining; out[4] = r->paint; out[5] = r->debt;
  return 0;
}
void b2v_ref_enc_set_paintover(void* h, int trigger_frames, int qp) { enc_t* e = (enc_t*)h; e->paint_trigger = trigger_frames; e->paint_qp = qp; }
/* slices of IDR pictures: n > 0 macroblocks per slice inside a row, n < 0 slices of slice_rows whole rows as in P pictures, 0 = the default rule */
void b2v_ref_enc_set_idr_slice_mbs(void* h, int n) {
  enc_t* e = (enc_t*)h;
  e->seg_cols = n < 0 ? 0 : n == 0 ? auto_seg_cols(e->mbw, e->mbh) : n >= e->mbw ? e->mbw : n;
}
void b2v_ref_enc_set_paintover_burst(void* h, int burst_frames) { ((enc_t*)h)->paint_burst = burst_frames > 0 ? burst_frames : 1; }
/* striped mode: stripe_rows macroblock rows per band (a multiple of slice_rows); 0 = full frame.  Returns the band count or -1. */
int b2v_ref_enc_set_stripes(void* h, int stripe_rows) {
  enc_t* e = (enc_t*)h;
  if (stripe_rows <= 0 || stripe_rows >= e->mbh) { e->stripe_rows = 0; e->n_stripes = 1; return 1; }
  if (e->auto_rows) { e->slice_rows = stripe_rows; e->n_slices = (e->mbh + e->slice_rows - 1) / e->slice_rows; }   /* default: one slice per band */
  if (stripe_rows % e->slice_rows) return -1;
  const int n = (e->mbh + stripe_rows - 1) / stripe_rows;
  if (n > MAX_STRIPES) return -1;
  e->stripe_rows = stripe_rows; e->n_stripes = n;
  const int last_rows = e->mbh - (n - 1) * stripe_rows, crop_r = (e->cw - e->width) / 2;
  e->sps_band_len[0] = build_sps(e->sps_band[0], e->mbw, stripe_rows, crop_r, 0);
  e->sps_band_len[1] = build_sps(e->sps_band[1], e->mbw, last_rows, crop_r, (e->ch - e->height) / 2);
  memset(e->stripe_fn, 0, sizeof e->stripe_fn);
  return n;
}
/* byte offset, size and coded flag of every band of the last encoded picture (3 ints each); returns the band count */
int b2v_ref_enc_stripe_table(void* h, int32_t* out) {
  enc_t* e = (enc_t*)h;
  if (!e->stripe_rows) return 0;
  memcpy(out, e->stripe_tab, sizeof(int32_t) * 3 * e->n_stripes);
  return e->n_stripes;
}
size_t b2v_ref_enc_max_au(void* h) { enc_t* e = (enc_t*)h; return (size_t)e->mbw * e->mbh * 1024 + 4096 + 128 * MAX_STRIPES; }

/*
 * Encode one picture.  cur_nv12: coded_w x coded_h NV12.  rc_mode 0 = CBR (target_bits per frame,
 * controller above), 1 = constant QP (qp_fixed).  Returns the access-unit size written to `out`.
 */
int64_t b2v_ref_enc_encode(void* h, const uint8_t* cur_nv12, int idr, int rc_mode, int qp_fixed, int64_t target_bits, uint8_t* out) {
  enc_t* e = (enc_t*)h;
  int mbs = e->mbw * e->mbh;
  const int k = (int)(e->pic & 1);
  const struct rcfb used = e->fb[k];                         /* the controller state after picture pic-2 */
  const int qp = rc_frame_qp(e, &used, idr, rc_mode, qp_fixed, target_bits);
  e->cur ^= 1;
  e->pic_seg = idr ? e->seg_cols : 0;
  const int nsl = pic_n_slices(e);
  if (idr) { e->frame_num = 0; }
  /* phase A: analysis + reconstruction.  Intra: macroblocks of a slice are sequential (left/top
   * dependencies), slices are independent.  Inter: every macroblock is independent. */
  if (idr) {
#pragma omp parallel for schedule(dynamic, 1)
    for (int s = 0; s < nsl; s++) {
      int row0 = s * e->slice_rows, row1 = (s + 1) * e->slice_rows, x0 = 0, x1 = e->mbw;
      if (e->pic_seg) { const int segs = pic_segs(e); row0 = s / segs; row1 = row0 + 1; x0 = (s % segs) * e->pic_seg; x1 = x0 + e->pic_seg; if (x1 > e->mbw) x1 = e->mbw; }
      if (row1 > e->mbh) row1 = e->mbh;
      for (int mby = row0; mby < row1; mby++)
        for (int mbx = x0; mbx < x1; mbx++) encode_intra_mb(e, cur_nv12, mbx, mby, qp);
    }
  } else {
    /* anchors first (their vectors are candidates for the rest of their groups), then everybody else */
    for (int pass = 0; pass < 2; pass++) {
#pragma omp parallel for schedule(dynamic, 1)
      for (int mby = 0; mby < e->mbh; mby++)
        for (int mbx = 0; mbx < e->mbw; mbx++) if (is_anchor(e, mbx, mby) == (pass == 0)) encode_inter_mb(e, cur_nv12, mbx, mby, qp);
    }
  }
  /* phase B: entropy coding per slice, then concatenation */
  uint8_t* skip = (uint8_t*)calloc(mbs, 1);
  size_t per = (size_t)e->slice_rows * e->mbw * 1024 + 256;
  if (e->pic_seg) per = (size_t)e->pic_seg * 1024 + 256;
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
      const int s0 = e->pic_seg ? r0 * pic_segs(e) : r0 / e->slice_rows, s1 = e->pic_seg ? r1 * pic_segs(e) : (r1 + e->slice_rows - 1) / e->slice_rows;
      for (int s = s0; s < s1; s++) { memcpy(out + o, tmp + per * s, lens[s]); o += lens[s]; bits += sbits[s]; }
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
