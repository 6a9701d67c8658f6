// jpeg.h — interface between the session layer (b2v_api.cu) and the JPEG stripe encoder (jpeg.cu; CaptureSettings.output_mode = 0).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "b2v_internal.h"    // AuHeader, BandEntry, AuLayout: the access-unit container of the striped H.264 mode

namespace b2v {

struct JpegEncoder;

struct JpegConfig {
  int width, height;       // visible size
  int coded_w, coded_h;    // multiples of 16 (the CSC pads by replication)
  int stripe_rows;         // MCU rows (16 luma rows) per stripe; 0 or >= picture rows = one stripe
  int quality;             // CaptureSettings.jpeg_quality
  int paint_quality;       // CaptureSettings.paint_over_jpeg_quality
  int paint_trigger;       // unchanged pictures before a stripe is re-sent at paint_quality; 0 = off
};

int  jpeg_create(const JpegConfig* cfg, JpegEncoder** out);
void jpeg_destroy(JpegEncoder* e);
AuLayout jpeg_layout(const JpegEncoder* e);       // always banded: n_bands >= 1 stripes
// enqueue one picture (NV12 in the JFIF matrix, coded size) on `st`; the output buffer gets AuHeader | BandEntry[n_stripes] | the
// JFIF files of the delivered stripes back to back.  force_all: deliver every stripe (first picture, refresh request).
// Returns the number of kernel launches issued.
int  jpeg_encode(JpegEncoder* e, const uint8_t* cur_nv12, uint8_t* au, int force_all, cudaStream_t st);
const char* jpeg_last_error();

}  // namespace b2v
