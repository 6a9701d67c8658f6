// b2v_internal.h — shared declarations between the C-ABI (b2v_api.cu) and the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/b2video.h"

namespace b2v {

// ---- access-unit container: both encoders write it into HBM, the session's output thread reads it ----
// 64-byte record the pack kernel writes in front of the access unit in HBM; travels to the host
// with the first D2H chunk.
struct AuHeader {
  int32_t size;            // bytes of data following the header (and band table)
  int32_t qp;              // slice QP used
  int32_t is_idr;
  int32_t n_slices;
  int64_t total_bits;      // before emulation prevention
  int32_t next_qp;         // rate controller output for the next frame
  int32_t overflow;        // non-zero if a macroblock exceeded its scratch budget (must never happen)
  uint64_t csc_t0, csc_t1;  // %globaltimer stamps of the CSC launch of this picture (0 when timing is off)
  int32_t pad[4];
};
static_assert(sizeof(AuHeader) == 64, "AuHeader must be 64 bytes");

// banded output (striped H.264, JPEG stripes): one record per band right after the AuHeader (offsets relative to the first data byte)
struct BandEntry { int32_t off, size, coded, frame_num; };

// B2V_FLAG_QUALITY: one record per band (one for a full frame) in front of the first data byte, written by k_quality (quality.cu)
struct QualityEntry {
  long long sse[3];        // exact sums of (S - R)^2: Y, Cb, Cr
  long long ssim_q40;      // sum over the band's SSIM windows of round(ssim * 2^40)
  long long windows;       // SSIM windows counted
};
static_assert(sizeof(QualityEntry) == 40, "QualityEntry must be 40 bytes");

// shape of an encoder's access-unit buffers
struct AuLayout {
  size_t cap;              // bytes of one buffer
  int data_off;            // bytes in front of the first data byte: AuHeader [+ band table] [+ quality table] (+ slack for an in-place
                           // stripe header)
  int n_bands;             // band table entries; 0 = full frame, no band table
  int band_rows;           // macroblock rows (16 luma rows) per band; 0 when n_bands == 0
  int quality_off = 0;     // bytes from the AuHeader to the QualityEntry table (max(n_bands, 1) entries); 0 = no table
};

// k_quality: the measurement of one picture (DESIGN.md §5.11).  S = the coded picture, R = its reconstruction, both NV12 at
// coded_w x coded_h; records of band_px luma rows (the last one cut at dst_h), columns 0 .. dst_w - 1.
struct QualityParams {
  const uint8_t* src;      // S
  const uint8_t* recon;    // R
  int coded_w, coded_h, dst_w, dst_h;
  int band_px, n_bands;
  QualityEntry* out;       // n_bands records in the access-unit buffer
  QualityEntry* acc;       // n_bands zeroed accumulators; k_quality leaves them zeroed
  unsigned int* done;      // zeroed block counter; k_quality leaves it zeroed
};
// returns number of kernel launches issued (1)
int launch_quality(const QualityParams& q, cudaStream_t st);

// ---- colour conversion spec (DESIGN.md §3; BT.709 limited range, 14-bit coefficients) ----
constexpr int KYR = 2991, KYG = 10064, KYB = 1016;
constexpr int KUR = -1649, KUG = -5547, KUB = 7196;
constexpr int KVR = 7196, KVG = -6536, KVB = -660;

// per-destination-index bilinear tap: i0 | (i1-i0)<<15 in .x low 16 / bit 15.., weight in .y
struct Tap { int32_t i0; int32_t i1; int32_t f; int32_t pad; };

struct CscParams {
  const uint8_t* src;   // device; pixels in the byte order `fmt` names
  int src_w, src_h, src_stride;
  int dst_w, dst_h;     // visible (scaled) size
  int coded_w, coded_h; // output plane size (multiples of 16 for the encoder; == dst for csc-only)
  uint8_t* out_y;       // coded_h rows, pitch coded_w
  uint8_t* out_uv;      // coded_h/2 rows, pitch coded_w
  const Tap* tx;        // dst_w taps (null when 1:1)
  const Tap* ty;        // dst_h taps
  unsigned long long* ts; // null, or {min block-start, max block-end} %globaltimer stamps of this launch (B2V_FLAG_TIMING)
  int matrix;             // 0 = BT.709 limited range (H.264 path), 1 = JFIF full-range BT.601 (JPEG stripe path)
  int fmt;                // B2V_PIX_*: 4 bytes per pixel (BGRA, RGBA) or 3 (BGR, RGB); src and src_stride are multiples of 4 for the
                          // 4-byte orders
};

// CscParams plus where a source that is not packed 8-bit pixels keeps its samples (b2v_submit_tensor).  The 1:1 kernels of packed
// pixels go on taking the CscParams part alone.
struct CscSource : CscParams {
  int dtype = B2V_DT_U8;     // B2V_DT_*: what one element is
  int stride_x = 0;          // bytes between two columns
  long long stride_c = 0;    // bytes between two channels; 0: packed 8-bit pixels, read as `fmt` says, and the two fields above are
                             // unused.  Otherwise element (c, y, x) is at src + c * stride_c + y * src_stride + x * stride_x,
                             // `fmt` tells only whether channel 0 is blue (even) or red (odd), and src is aligned to the element
};

// returns number of kernel launches issued (1)
int launch_csc(const CscSource& p, cudaStream_t st);
void make_taps_host(Tap* t, int dn, int sn);
// B2V_FLAG_DAMAGE (csc.cu): rectangles -> dirty-tile map of ceil(dst_w / 16) x ceil(dst_h / 16) bytes; returns the dirty count.
// tx / ty: the host taps of the scale, null at 1:1.  Rectangles are checked by the caller.
int damage_tiles(const Tap* tx, const Tap* ty, int src_w, int src_h, int dst_w, int dst_h, const b2v_rect* rects, int n, uint8_t* map);
// converts only the n tiles listed in d_tiles (ty * ceil(dst_w / 16) + tx each), one launch even for n == 0; returns 1
int launch_csc_tiles(const CscSource& p, const int* d_tiles, int n, cudaStream_t st);

}  // namespace b2v
