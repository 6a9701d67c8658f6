// h264_encoder.h — interface between the session layer (b2v_api.cu) and the H.264 Baseline
// encoder kernels (h264_*.cu).  H100 carries no NVENC block, so stage (c) of the hot path is a
// software encoder made of CUDA kernels: one warp per macroblock.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "b2v_internal.h"

namespace b2v {

struct Encoder;

struct EncoderConfig {
  int width, height;       // visible size (SPS cropping)
  int coded_w, coded_h;    // multiples of 16
  int slice_rows;          // macroblock rows per slice
  int stripe_rows;         // macroblock rows per band (multiple of slice_rows); 0 = full-frame
  int idr_slice_mbs;       // IDR pictures, whatever slice_rows is: macroblocks per slice inside a row; 0 = default rule (>= 0)
  int flags;               // the session's B2V_FLAG_*, a combination check_coding_flags (b2v_api.cu) allows.  The encoder reads:
                           //   B2V_FLAG_QUALITY: k_quality measures every band into the access unit's quality table
                           //   B2V_FLAG_DROPPABLE: every P picture at an odd count from the IDR is a non-reference picture
                           //   B2V_FLAG_WIDE_MOTION: coarse vectors per anchor group (k_coarse) and windows centred on far candidates
                           //   B2V_FLAG_LONG_TERM_REF: one long-term reference picture, marked on the GPU (k_ltr_mark)
                           //   B2V_FLAG_SIZE_CAP: P pictures over max_picture_bytes coded again at a coarser QP (k_size_cap)
};

struct EncodeFrameParams {
  const uint8_t* cur;      // NV12, coded size, device
  uint8_t* au;             // device buffer, encoder_layout().cap bytes; AuHeader first
  int idr;
  int rc_mode;             // B2V_RC_CBR | B2V_RC_CQP
  int qp_fixed;
  int paint_trigger, paint_qp, paint_burst;   // paint-over: `paint_burst` pictures at paint_qp after `paint_trigger` all-skipped pictures (0 = off)
  int64_t target_bits;     // per frame, CBR
  cudaEvent_t* ev;         // null, or 6 timing events: encoder records ev[2..5] after each stage (forces the serial schedule)
  int max_picture_bytes;   // B2V_FLAG_SIZE_CAP: this picture's cap (0 = none)
  cudaStream_t st_pack;    // null = everything on `st` (always with B2V_FLAG_SIZE_CAP); else the entropy coding of this picture (k_cavlc_mb ... k_pack_au) runs here,
                           // overlapping the analysis of the next picture on `st`.  The access unit is complete on st_pack.
  const unsigned long long* csc_ts;   // null, or the CSC launch's device stamps to forward in the AuHeader
};

int  encoder_create(const EncoderConfig* cfg, Encoder** out);
void encoder_destroy(Encoder* e);
AuLayout encoder_layout(const Encoder* e);       // n_bands == 0 when full-frame
// enqueue one frame on `st` (and `p->st_pack`); returns the number of kernel launches issued
int  encoder_encode(Encoder* e, const EncodeFrameParams* p, cudaStream_t st);
const uint8_t* encoder_recon(const Encoder* e);   // NV12 reconstruction of the last encoded frame
const char* encoder_last_error();

}  // namespace b2v
