/*
 * b2video.h — C-ABI of libb2video.so, the H100-native (sm_90a) video-frame hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  Every entry point replaces one
 * call the selkies reference makes into its out-of-tree native module
 * `pixelflux` (capture → colour-convert → H.264 encode → callback).  The
 * reference interface each entry replaces is cited as  path:line  relative to
 * the selkies tree.  The signatures carry plain pointers and sizes only; the
 * Python host side (selkies_b200/_native.py) binds them with ctypes.
 *
 * Threading: every function is safe to call from any host thread; setters may
 * race with b2v_ring_submit() (reference: control calls arrive on thread-pool
 * threads, media_pipeline.py:195,236,244,300,313).  b2v_set_resolution() locks
 * submitters out, drains, and returns B2V_ESTATE while a producer still holds an
 * acquired ring slot (its memory is about to be reallocated).  The frame callback fires on
 * the session's own output thread (a native, non-Python thread, as pixelflux's
 * does: media_pipeline.py:293 uses run_coroutine_threadsafe for that reason).
 *
 * Errors: functions returning int give 0 on success and a negative B2V_E* code
 * on failure; b2v_last_error() returns a thread-local message.
 */
#ifndef B2VIDEO_H_
#define B2VIDEO_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2V_ABI_VERSION 4

enum {
  B2V_OK = 0,
  B2V_EINVAL = -1,   /* bad argument / unsupported size            */
  B2V_ECUDA = -2,    /* CUDA runtime error (see b2v_last_error)     */
  B2V_ENOMEM = -3,
  B2V_ESTATE = -4,   /* call not valid in the current state         */
  B2V_ETIMEOUT = -5
};

/* rate-control modes: reference CaptureSettings.h264_cbr_mode / h264_crf
 * (media_pipeline.py:266-269) */
enum { B2V_RC_CBR = 0, B2V_RC_CQP = 1 };

/* header_mode: what precedes the Annex-B access unit in b2v_frame.data.
 * 1 = the 10-byte pixelflux stripe header the reference strips at
 * media_pipeline.py:286 and keeps at selkies.py:3116
 * (0x04, frame_type, frame_id u16be, y_start u16be, width u16be, height u16be;
 * parser: addons/selkies-web-core/selkies-ws-core.js:3183-3196). */
enum { B2V_HDR_NONE = 0, B2V_HDR_PIXELFLUX = 1 };

/* Session configuration — the native image of pixelflux.CaptureSettings as
 * filled by MediaPipelinePixel.generate_capture_settings
 * (media_pipeline.py:251-273) and _get_capture_settings (selkies.py:3191-3242). */
typedef struct b2v_settings {
  int32_t src_w, src_h;     /* BGRA source size (even, 16..7680 x 16..4320; selkies.py:281) */
  int32_t dst_w, dst_h;     /* encoded size; 0 = same as source (no scaling)                */
  double  fps;              /* CaptureSettings.target_fps                                   */
  int32_t device;           /* CUDA ordinal (settings.py:162 gpu_id)                        */
  int32_t rc_mode;          /* B2V_RC_CBR | B2V_RC_CQP                                      */
  int32_t bitrate_kbps;     /* CaptureSettings.h264_bitrate_kbps                            */
  int32_t crf;              /* CaptureSettings.h264_crf → constant QP 0..51 in CQP mode; <0 = 26 */
  int32_t gop;              /* in FRAMES.  <=0: IDR only on request (settings.py:163 keyframe_distance=-1);
                               1: intra-only; N: IDR every N frames.  keyframe_distance itself is in SECONDS:
                               the host side passes round(seconds * fps) (pixelflux_compat.py)             */
  int32_t slice_rows;       /* macroblock rows per slice of a P picture (>=1); 0 = default: 8, or one slice per stripe in striped
                               mode (inside a slice P_Skip infers moving vectors: a scrolling picture costs half the bytes) */
  int32_t header_mode;      /* B2V_HDR_*                                                    */
  int32_t ring_slots;       /* pinned BGRA ingest ring depth (2..16); 0 = default 4          */
  int32_t flags;            /* B2V_FLAG_*                                                   */
  int32_t paintover_trigger_frames; /* after this many consecutive all-skipped pictures code paintover_burst_frames pictures
                                       at paintover_crf (CaptureSettings.paint_over_trigger_frames / use_paint_over_quality,
                                       selkies.py:3226-3229); in CBR mode the paint-over QP only applies when it is finer
                                       than the controller's; 0 = off */
  int32_t paintover_crf;            /* CaptureSettings.h264_paintover_crf */
  int32_t stripe_rows;      /* striped mode (CaptureSettings.h264_fullframe = False, selkies.py:3219; encoder
                               "x264enc-striped"): macroblock rows per stripe, a multiple of slice_rows.  Every stripe is
                               an independent H.264 stream (own SPS/PPS, own frame_num, motion confined to the stripe)
                               delivered by its own callback with y_start/height (10-byte header bytes 4..9,
                               selkies-ws-core.js:3183-3196); a stripe whose macroblocks were all skipped is not
                               delivered.  0 or >= picture rows = full frame */
  int32_t idr_slice_mbs;    /* IDR pictures only (whatever slice_rows is): macroblocks per slice INSIDE a row.  The macroblocks of an
                               intra slice are a serial chain (left-neighbour prediction), so shorter slices shorten the chain the
                               GPU has to walk.  0 = default (about 540 slices per picture, none under 30 macroblocks: 60 at 4K,
                               30 at 1080p), n > 0 = n macroblocks per slice (n >= the picture's width in macroblocks: one slice
                               per row).  Negative values are rejected: b2v_create fails with B2V_EINVAL.  (Earlier builds of
                               this ABI version took a negative value to mean slices of whole rows.) */
  int32_t paintover_burst_frames;   /* CaptureSettings.h264_paintover_burst_frames (selkies.py:3217): how many consecutive
                                       pictures are coded at paintover_crf once the trigger is reached; <= 0 = 1 */
} b2v_settings;

enum {
  B2V_FLAG_SPS_EVERY_IDR = 1,   /* in-band SPS/PPS before every IDR (rtc.py:394-401); always on */
  B2V_FLAG_NO_ENCODE     = 2,   /* CSC only (BASELINE config 4: 8K CSC roofline stress)         */
  B2V_FLAG_TIMING        = 4,   /* bracket every kernel with CUDA events (b2v_get_stats)        */
  B2V_FLAG_DEVICE_TIMER  = 8,   /* with TIMING: the CSC kernel also stamps %globaltimer (ms_csc_device) */
  B2V_FLAG_TIMING_CSC    = 16,  /* a CUDA-event pair around the CSC launch of every 4th picture (ms_csc / n_csc)  */
  B2V_FLAG_JPEG          = 32,  /* CaptureSettings.output_mode = 0 (selkies.py:3209-3212): JPEG stripes instead of H.264.  The picture is cut
                                   into stripes of stripe_rows x 16 rows (0 = about eight stripes); each stripe that changed is delivered by its
                                   own callback as one baseline JFIF file (JFIF colour, 4:2:0), y_start/height set; with B2V_HDR_PIXELFLUX the
                                   file is preceded by frame_id u16be | y_start u16be (the reference adds 03 00 in front, selkies.py:3118).
                                   crf = jpeg_quality, paintover_crf = paint_over_jpeg_quality, paintover_trigger_frames as for H.264.
                                   A key-frame request re-sends every stripe. */
  B2V_FLAG_QUALITY       = 64,  /* measure every delivered record on the GPU (b2v_frame_quality): SSE per plane and luma SSIM of the
                                   reconstruction against the picture the encoder coded.  H.264 only: b2v_create rejects it with
                                   B2V_FLAG_JPEG or B2V_FLAG_NO_ENCODE (B2V_EINVAL), which have no reconstruction.  The access units
                                   are the same bytes with and without it; it costs one kernel launch per picture (kernel_launches). */
  B2V_FLAG_DROPPABLE     = 128, /* two temporal layers, so that a consumer that falls behind can shed pictures without corrupting the
                                   stream.  The pictures of a session are counted from each IDR (the IDR is 0; b2v_request_idr,
                                   gop and b2v_set_resolution restart the count).  Every P picture at an odd count is a
                                   non-reference picture: all its slices have nal_ref_idc = 0 and no dec_ref_pic_marking().  Every
                                   other picture is a reference picture, as without the flag.  A P picture at an even count
                                   predicts from the reference picture two before it, one at an odd count from the picture just
                                   before it.  frame_num advances by one after each reference picture only: a non-reference picture
                                   carries the frame_num of the reference picture that follows it.  The SPS does not change
                                   (max_num_ref_frames 1, no frame_num gaps).  A consumer may drop any set of non-reference access
                                   units; the rest decodes to exactly the encoder's reconstructions of the pictures it kept.  It
                                   tells a droppable access unit by the NAL header byte of its first slice (nal_ref_idc, bits 5..6,
                                   is 0).  b2v_get_recon returns the last coded picture, droppable or not.  H.264 full-frame only:
                                   b2v_create rejects it (B2V_EINVAL) with B2V_FLAG_JPEG, B2V_FLAG_NO_ENCODE or in striped mode
                                   (stripe_rows > 0 and less than the picture's macroblock rows), and b2v_set_resolution rejects a
                                   size at which stripe_rows would stripe.  It costs a third reconstruction buffer (coded
                                   width x height x 1.5 bytes). */
  B2V_FLAG_WIDE_MOTION   = 256, /* find motion vectors beyond the +-16 samples of the P-picture search, for fast scrolls and window
                                   drags.  Every picture gets a 1/4 x 1/4 decimated luma plane; in every 4 x 4-macroblock group
                                   whose anchor's co-located block changed, that block is searched in the reference picture's
                                   plane over +-128 samples horizontally and +-256 vertically, inside the picture and the band.
                                   The anchor then also searches +-16 samples around that coarse vector, and a temporal or anchor
                                   predictor beyond the co-located window is tested in a window centred on it.  Every vector
                                   component stays within [-256, 255.75] samples, the range the SPS's VUI asserts.  The SPS and
                                   the syntax do not change; the access units do (that is the point).  Works with stripes,
                                   scaling, B2V_FLAG_DROPPABLE and B2V_FLAG_QUALITY.  H.264 only: b2v_create rejects it
                                   (B2V_EINVAL) with B2V_FLAG_JPEG or B2V_FLAG_NO_ENCODE.  It costs one kernel launch per picture
                                   (kernel_launches) and coded width x height / 16 bytes per reconstruction buffer. */
  B2V_FLAG_LONG_TERM_REF = 512, /* keep one earlier picture as a long-term reference, so that content that comes back (a popup or
                                   menu closing, a switch back to an application, a window dragged off the desktop) is predicted
                                   from it instead of coded as new.  The SPS says max_num_ref_frames 2 and max_dec_frame_buffering 2.
                                   P picture k marks picture k-1 long-term (adaptive dec_ref_pic_marking: MMCO 4, MMCO 3 with
                                   long_term_frame_idx 0, preceded by MMCO 1 on the picture two back while no long-term picture
                                   exists) when changed(k) >= max(ceil(macroblocks / 64), 8 x changed(k-1)), changed being the count
                                   of macroblocks whose co-located block fails the zero-motion exit (an IDR counts all); every other
                                   P picture uses the sliding window.  The GPU decides it per picture.  While a long-term picture
                                   exists, P slices have two active references (the previous picture, then the long-term one) and a
                                   macroblock whose zero vector into the long-term picture is within the zero-motion threshold is
                                   coded from it (P_L0_16x16, ref_idx_l0 1, zero vector).  An IDR (requested, gop or
                                   b2v_set_resolution) clears it.  Works with CQP and CBR, paint-over, scaling, cropping,
                                   B2V_FLAG_QUALITY and B2V_FLAG_WIDE_MOTION.  H.264 full-frame only: b2v_create rejects it
                                   (B2V_EINVAL) with B2V_FLAG_JPEG, B2V_FLAG_NO_ENCODE, B2V_FLAG_DROPPABLE or in striped mode, and
                                   b2v_set_resolution rejects a size at which stripe_rows would stripe.  It costs one kernel launch
                                   per P picture (kernel_launches), a copy of one picture on the pictures that mark, and coded
                                   width x height x 1.5 bytes. */
  B2V_FLAG_DAMAGE        = 1024,/* damage rectangles (an ingest flag, not a coding flag: it works with H.264 full-frame and striped,
                                   B2V_FLAG_JPEG, B2V_FLAG_NO_ENCODE and every coding flag).  The b2v_*_damage submits take the
                                   regions of the source that changed since the previous picture; only those are copied and
                                   colour-converted.  The contract: when the rectangles cover every pixel that changed since the
                                   previous picture of the session, the access units, the reconstructions and the NV12 pictures are
                                   exactly those of a whole-frame submit of the same picture.  The ring then copies into one
                                   persistent device frame (the mirror, src_w x src_h x 4 bytes) instead of one device buffer per
                                   ring slot: at 4K that is 33 MB of HBM instead of ring_slots x 33 MB. */
  B2V_FLAG_SCENE_CUT     = 2048,/* scene cuts: a P picture whose content is all new (an application switch, a slide change, a cut in a
                                   video) is coded as an intra picture instead of predicted from a picture it no longer resembles.
                                   The GPU decides per P picture, after the P analysis, which runs unchanged:
                                     cost_inter = the sum over macroblocks of the luma cost of the prediction the analysis chose:
                                                  SAD + lambda(QP) x (se(v) bits of both vector components, + 4 when the vector is
                                                  fractional), a long-term macroblock counting the zero vector's bits, and 0 for a
                                                  macroblock whose SAD is at most 96 x lambda(QP) (the zero-motion exit's threshold:
                                                  its residual is quantisation noise); while a long-term picture is a reference, the
                                                  smaller of that and the same cost of the long-term picture's zero vector, for every
                                                  macroblock, so that content that comes back stays P;
                                     cost_intra = the sum over macroblocks of the smallest luma SAD of Intra16x16 vertical,
                                                  horizontal and DC prediction from the SOURCE picture's neighbouring samples
                                                  (neighbours outside the picture unavailable, 8.3.3; slices ignored), + 16 x
                                                  lambda(QP) per macroblock;
                                     the picture is cut when cost_intra < cost_inter (lambda: the motion-search table, DESIGN.md §5.3).
                                   A cut picture is a non-IDR intra picture: NAL type 1, every slice of slice_type 7, in the IDR
                                   slice grid (idr_slice_mbs), at the QP the P picture would have had, with the frame_num,
                                   nal_ref_idc and dec_ref_pic_marking() the P picture would have had; its macroblocks are coded by
                                   the intra coder of IDR pictures.  It carries no parameter sets, is_key stays 0, the gop count,
                                   the droppable layers and the long-term picture go on as after a P picture, and the SPS does not
                                   change.  The next picture predicts from its reconstruction and finds no temporal predictor in it,
                                   as after an IDR.  A consumer tells a cut picture by the slice_type of its first slice
                                   (h264_nal.is_intra).  Works with CQP and CBR, paint-over, scaling, cropping, B2V_FLAG_QUALITY,
                                   B2V_FLAG_WIDE_MOTION, B2V_FLAG_DROPPABLE, B2V_FLAG_LONG_TERM_REF (whose long-term candidate is
                                   part of cost_inter) and B2V_FLAG_DAMAGE.  H.264 full-frame only: b2v_create rejects it
                                   (B2V_EINVAL) with B2V_FLAG_JPEG, B2V_FLAG_NO_ENCODE or in striped mode, and b2v_set_resolution
                                   rejects a size at which stripe_rows would stripe.  It costs two kernel launches per P picture
                                   (kernel_launches: k_scene_cut, and k_intra_rows, which returns at once unless the picture was
                                   cut), flagged variants of the analysis and entropy kernels, and 4 bytes per macroblock. */
  B2V_FLAG_SIZE_CAP      = 4096 /* picture size cap: a P picture larger than b2v_set_max_picture_bytes is coded once more at a
                                   coarser QP, decided on the GPU with no host round trip.  In a low-latency stream the size of a
                                   picture is the time it holds the link; this bounds the spikes the CBR controller (which feeds
                                   back two pictures late and repays a spike afterwards) lets through.
                                     size: the sum of the picture's macroblock-layer bits (mb_type to the last residual block of
                                           every coded macroblock; an I_PCM macroblock's mb_type and 384 samples), rounded up to
                                           bytes.  Slice headers, mb_skip_run, I_PCM alignment bits (at most 7 per macroblock),
                                           parameter sets, start codes and emulation-prevention bytes are not counted.
                                     rule:  when size > cap, the picture is coded again once at QP' = QP + d, d the smallest value in
                                           1..51-QP with bits <= (8 x cap x T[d]) >> 16, T[d] = round(65536 x 2^(d/6)) (integers
                                           only); 51 when none qualifies.  A picture at QP 51 is not recoded.
                                   There is one recode and no second pass: the cap is a target, and a recoded picture can still
                                   exceed it (the rule assumes bits halve every 6 QP steps).  A recode keeps the analysis's vectors,
                                   reference indices and exits; every macroblock gets the same motion-compensated prediction and a
                                   new residual at QP' (transform, quantisation, reconstruction, levels); P_Skip and the I_PCM
                                   fallback are decided again on the new levels, in both directions.  Every slice's slice_qp_delta
                                   carries QP', b2v_frame.qp reports it, and the CBR controller and the paint-over scheduler see
                                   the picture as finally coded.  Only P pictures are capped (the macroblocks coded from the
                                   long-term picture included); IDR pictures and scene-cut intra pictures are not.  In striped mode
                                   the cap applies to the whole access unit, all bands together (the QP is the picture's).
                                   With cap 0 (the default) the flag changes no output byte.  Works with CQP and CBR, paint-over,
                                   scaling, cropping, striped mode and every other coding flag.  H.264 only: b2v_create rejects it
                                   (B2V_EINVAL) with B2V_FLAG_JPEG or B2V_FLAG_NO_ENCODE.  It costs three kernel launches per P
                                   picture (kernel_launches: k_size_cap, k_requant and a second CAVLC pass, which return at once
                                   unless the picture is recoded), 388 bytes per macroblock, and the overlap of a picture's entropy
                                   coding with the next picture's analysis: a recode rewrites the reconstruction the next picture
                                   predicts from, so entropy coding runs on the analysis stream. */
};

/* B2V_FLAG_DAMAGE: one changed region of the source, in source pixels of the frame (or the device window) the submit names.
 * Rectangles are clipped to the frame; w == 0 or h == 0 is an empty rectangle. */
typedef struct b2v_rect { int32_t x, y, w, h; } b2v_rect;
#define B2V_MAX_DAMAGE_RECTS 64    /* most rectangles of one submit (each ring rectangle is one copy); merge beyond it */

/* One encoded frame, the native image of the pixelflux callback result
 * (`result.data / result.size / result.frame_id`, media_pipeline.py:284-292).
 * `data` is owned by the library and valid only during the callback. */
typedef struct b2v_frame {
  const uint8_t* data;   /* [optional 10-byte header] + Annex-B access unit */
  int32_t  size;         /* bytes in data                                    */
  int32_t  frame_id;     /* +1 per emitted frame, wraps at 65536 (selkies.py:10) */
  int32_t  is_key;       /* 1 = IDR                                         */
  int32_t  qp;           /* slice QP used for this frame                     */
  int64_t  pts90k;       /* frame_id * (90000 // fps)  (media_pipeline.py:291-292) */
  int64_t  capture_ns;   /* value passed to b2v_ring_submit                  */
  int32_t  y_start;      /* first picture row of this stripe (0 when full-frame)           */
  int32_t  height;       /* visible rows in this stripe (the picture height when full-frame) */
} b2v_frame;

typedef void (*b2v_cb)(const b2v_frame* frame, void* user);

/* B2V_FLAG_QUALITY: the measurement of one delivered record (the whole picture in full-frame mode, one band in striped mode).
 * S is the NV12 picture the encoder coded (after colour conversion and scaling), R its reconstruction, which is what a decoder
 * outputs.  Both are taken on the record's rows y_start .. y_start + height - 1 and columns 0 .. dst_w - 1; chroma on rows
 * y_start / 2 .. and half the width.  Padding below or right of the visible picture is never counted.
 *   sse_*: exact sums of (S - R)^2 per plane; samples_y = dst_w * height, samples_c = samples_y / 4.
 *   PSNR of a plane = 10 log10(255^2 * samples / sse) (infinite when sse is 0).
 *   ssim_y (luma): the mean over the 8x8 windows whose origins lie on a 4-sample grid anchored at (0, y_start) and that lie
 *   wholly inside the record.  Per window, over its 64 samples: Sx = sum s, Sy = sum r, Q = sum (s^2 + r^2), P = sum s*r,
 *   V = 64 Q - Sx^2 - Sy^2, C = 64 P - Sx Sy (exact integers), and in IEEE fp64 (the four factors converted, the two products
 *   formed, then one division):
 *     ssim = ((2 Sx Sy + 416) (2 C + 235963)) / ((Sx^2 + Sy^2 + 416) (V + 235963))
 *   (416 = round(0.01^2 255^2 64), 235963 = round(0.03^2 255^2 64 63), as x264 --ssim).  ssim_windows counts the windows;
 *   when it is 0 (a record with fewer than 8 rows or columns) ssim_y is NaN.  The mean is exact to within 2^-41: each window's
 *   value is summed as round(ssim * 2^40) in int64, so the result does not depend on the order of summation. */
typedef struct b2v_quality {
  int64_t sse_y, sse_cb, sse_cr;
  int64_t samples_y, samples_c;
  double  ssim_y;
  int64_t ssim_windows;
} b2v_quality;

/* Per-session counters; kernel times are CUDA-event milliseconds accumulated on
 * the launching stream (only when B2V_FLAG_TIMING is set). */
typedef struct b2v_stats {
  int64_t frames_submitted, frames_delivered, key_frames;
  int64_t bytes_out, h2d_bytes, d2h_bytes;
  int64_t kernel_launches;
  double  ms_csc, ms_intra, ms_inter, ms_cavlc, ms_slice, ms_pack, ms_total_gpu;
  int64_t n_csc, n_intra, n_inter, n_cavlc, n_slice, n_pack;
  double  ms_csc_device;   /* same launches, timed by the kernel itself (%globaltimer: first block start .. last block end) */
  int64_t n_csc_device;
  /* host-side stopwatches (CLOCK_MONOTONIC ns, always on): where a session's wall time goes when it is not the GPU's */
  int64_t ns_wait_event;     /* output thread: waiting for the GPU to finish the next picture (polling, no interrupt)      */
  int64_t ns_wait_event_max; /*   longest single such wait                                                               */
  int64_t n_event_sleeps;    /*   waits that outlasted the 30 us busy phase and slept                                    */
  int64_t ns_wait_job;       /* output thread: idle, no picture in flight                                                */
  int64_t ns_callback;       /* output thread: inside the frame callback (Python holds the GIL there)                    */
  int64_t ns_wait_out_slot;  /* submitter: blocked on back-pressure (every output slot in flight)                        */
  int64_t ns_wait_ring;      /* producer: blocked in b2v_ring_acquire (every ingest slot in flight)                      */
  int64_t ns_submit;         /* submitter: inside the CUDA enqueue calls of a picture (launches, copies, event records)  */
} b2v_stats;

/* ---- lifecycle: replaces ScreenCapture() / start_capture / stop_capture
 *      (media_pipeline.py:298-300, 313; selkies.py:3163-3176, 2852) ---------- */
int  b2v_abi_version(void);
int  b2v_device_count(void);
int  b2v_create(const b2v_settings* s, b2v_cb cb, void* user, void** out_handle);
void b2v_destroy(void* h);                 /* blocks: drains frames, joins the output thread */

/* ---- frame ingest (a: pinned host ring → cudaMemcpyAsync).  The producer is
 *      whatever fills BGRA frames (pixelflux's XShm grab in the reference,
 *      SURVEY.md §3.2 hot loop #1). ------------------------------------------ */
void* b2v_ring_acquire(void* h, int32_t* slot);          /* blocks until a slot is free */
int   b2v_ring_submit(void* h, int32_t slot, int32_t stride_bytes, int64_t capture_ns);
/* Give an acquired slot back WITHOUT encoding it (the producer had no frame after all: end of a canned source, a grab that
 * failed).  Only the most recently acquired slot can be returned; the next b2v_ring_acquire hands out the same slot. */
int   b2v_ring_release(void* h, int32_t slot);
/* device-resident frames (bench `value`: inputs already in HBM); b2v_submit_resident is b2v_submit_device of the library's own
 * copy (BGRA, no producer stream) */
int   b2v_resident_upload(void* h, int32_t index, const void* bgra_host, int32_t stride_bytes);
int   b2v_submit_resident(void* h, int32_t index, int64_t capture_ns);

/* ---- frame ingest from device memory (a producer whose frames are already on the session's GPU: a renderer through CUDA/GL
 *      interop, a compositor's exported buffers; for a PyTorch model's tensors see b2v_submit_tensor).  No copy: the colour
 *      conversion reads the frame in place. */
enum { B2V_PIX_BGRA = 0, B2V_PIX_RGBA = 1, B2V_PIX_BGR = 2, B2V_PIX_RGB = 3 };   /* byte order in memory; alpha ignored */
/* Encodes `frame`: src_h rows of src_w pixels (the session's source size; scaling, striped mode, JPEG mode and
 * B2V_FLAG_NO_ENCODE apply as for b2v_ring_submit) at `pitch_bytes`, in device (or managed) memory of the session's GPU.
 *
 * Stream order, both ways.  `cuda_stream` is the producer's stream on the session's device (NULL = the legacy default stream;
 * cudaStreamPerThread is accepted).  The picture's colour conversion runs after everything enqueued on `cuda_stream` before this
 * call (an event recorded there, waited on by the library's stream: the host never blocks on the producer), and work enqueued
 * on `cuda_stream` after this call runs after that conversion (an event recorded behind it, waited on by `cuda_stream`).  So
 * when the call returns, the producer may overwrite or free the buffer in stream order on `cuda_stream`; from another stream it
 * must order itself after `cuda_stream` first.  Settings apply as for any submit (see "When a call takes effect" below).
 *
 * Rejections (B2V_EINVAL + message, nothing enqueued, the session keeps running): an unknown pixel_format; a null handle or
 * frame; pitch_bytes < src_w * bytes per pixel; frame or pitch not a multiple of 4 for BGRA / RGBA; memory that is not device
 * or managed memory of the session's device (host memory, pinned and mapped host memory included: the kernel would read it
 * over PCIe); a frame whose last byte, frame + pitch_bytes * (src_h - 1) + src_w * bytes per pixel - 1, lies outside the
 * allocation that holds `frame`.  A stream of another device fails the session like any CUDA error during a submit. */
int   b2v_submit_device(void* h, const void* frame, int32_t pitch_bytes, int32_t pixel_format, void* cuda_stream, int64_t capture_ns);

/* ---- frame ingest of a device tensor as a model leaves it: planar or interleaved, uint8 or floating point in [0, 1], any strides.
 *      No preparation pass: the colour conversion reads the elements where they are and quantises them in registers. */
enum { B2V_DT_U8 = 0, B2V_DT_F16 = 1, B2V_DT_BF16 = 2, B2V_DT_F32 = 3 };
typedef struct b2v_tensor {
  const void* data;                       /* element (channel 0, row 0, column 0) of the src_w x src_h picture */
  int32_t dtype;                          /* B2V_DT_*                                                         */
  int32_t pixel_format;                   /* B2V_PIX_*: how many channels (BGRA / RGBA 4, BGR / RGB 3; a fourth is never read) and
                                             whether channel 0 is blue or red                                 */
  int64_t stride_c, stride_y, stride_x;   /* bytes; each positive and a multiple of the element size: the element of channel c,
                                             row y, column x is at data + c * stride_c + y * stride_y + x * stride_x.  One
                                             description for (C, H, W), (H, W, C), channels_last, a slice of a batch, a window
                                             of a larger surface and a padded pitch */
} b2v_tensor;
/* b2v_submit_device with this richer description of the frame: the same stream order both ways (the producer may overwrite the
 * tensor in stream order on `cuda_stream` when the call returns), the same settings, scaling and modes.
 *
 * Element -> 8-bit sample: uint8 is the value; fp16 / bf16 / fp32 widen to fp32 and give
 * q = round_half_even(255 * min(max(x, 0), 1)), one fp32 multiplication; NaN -> 0, -0 -> 0, +inf -> 255 (DESIGN.md §3).  The three
 * samples of a pixel then take the integer colour conversion of every other entry.  Other value ranges are the caller's to map.
 *
 * Rejections (B2V_EINVAL + message, nothing enqueued, the session keeps running): a null handle, descriptor or data; an unknown
 * dtype or pixel_format; a stride that is <= 0, not a multiple of the element size, or too large (stride_y, stride_x: 2^31 and up;
 * stride_c: 2^48 and up); data not
 * aligned to the element size; memory that is not device or managed memory of the session's device; a last byte read,
 * data + 2 * stride_c + (src_h - 1) * stride_y + (src_w - 1) * stride_x + element size - 1, outside the allocation holding `data`. */
int   b2v_submit_tensor(void* h, const b2v_tensor* t, void* cuda_stream, int64_t capture_ns);

/* ---- damage submits (B2V_FLAG_DAMAGE).  b2v_ring_submit, b2v_submit_device and b2v_submit_tensor are these with rects = NULL.
 *   rects == NULL: the whole frame.  n_rects == 0 with rects != NULL: nothing changed; the picture is still coded and delivered.
 *   Rejections (B2V_EINVAL, before any CUDA call; a ring slot stays acquired): rects without B2V_FLAG_DAMAGE, a negative w or h,
 *   n_rects < 0 or above B2V_MAX_DAMAGE_RECTS, a null handle.
 * Ring: copies exactly the given rectangles of the slot into the mirror, one 2-D copy each, so the producer only has to write
 *   those rectangles into the slot.  A damage submit needs the previous picture of the session to be a ring picture at the
 *   current geometry: otherwise (the first picture after b2v_create or b2v_set_resolution, a ring picture after a device,
 *   tensor or resident picture) it fails with B2V_ESTATE and the slot stays acquired, so the producer can fill it whole and
 *   submit it again.  A whole-frame ring submit of a flagged session copies the whole slot into the mirror.  The copy of a
 *   picture waits for the colour conversion of the one before to have read the mirror.
 * Device and tensor: the frame is read in place, so there is no copy to save; only the tiles the rectangles touch are converted.
 *   With no previous picture at this geometry the whole frame is converted.
 * The conversion: the rectangles are mapped to 16 x 16 tiles of the coded picture (b2v_damage_tiles); when the dirty tiles cover
 *   more than a quarter of the picture (DESIGN.md §4, damage rectangles), and for whole-frame submits, the whole frame is converted as without the
 *   flag.  Either way one CSC kernel per picture (kernel_launches).  stats.h2d_bytes counts the pixel bytes actually copied:
 *   4 x the clipped rectangle area of a ring damage submit, src_w x src_h x 4 of a whole one. */
int   b2v_ring_submit_damage(void* h, int32_t slot, int32_t stride_bytes, const b2v_rect* rects, int32_t n_rects, int64_t capture_ns);
int   b2v_submit_device_damage(void* h, const void* frame, int32_t pitch_bytes, int32_t pixel_format, const b2v_rect* rects,
                               int32_t n_rects, void* cuda_stream, int64_t capture_ns);
int   b2v_submit_tensor_damage(void* h, const b2v_tensor* t, const b2v_rect* rects, int32_t n_rects, void* cuda_stream, int64_t capture_ns);
int   b2v_flush(void* h);                               /* wait until every submitted frame was delivered */

/* ---- live control: ScreenCapture.update_framerate (media_pipeline.py:236),
 *      update_video_bitrate (:195), request_idr_frame (:244); set_resolution is
 *      WebRTCApp.on_resize_handler → width/height (webrtc_mode.py:383-426).
 * When a call takes effect: every setting is read when a picture is submitted, so a control call made after submit k and
 * before submit k+1 applies from picture k+1 on, whether or not pictures are still in flight; nothing already submitted
 * changes.  b2v_request_idr makes picture k+1 an IDR; with b2v_set_gop(frames > 0), picture k+1 is an IDR when
 * `frames` or more pictures, the last IDR included, were coded since that IDR.  b2v_set_resolution first drains the pictures in flight, then restarts the encoder:
 * picture k+1 is an IDR with parameter sets of the new size, the rate controller starts afresh, frame ids continue.  In CBR
 * mode the controller sees a new bitrate or frame rate as a new per-picture target (bitrate * 1000 / fps bits); its QP
 * decisions reach the pictures two after the one they were made from. --- */
int  b2v_set_framerate(void* h, double fps);
int  b2v_set_bitrate_kbps(void* h, int32_t kbps);
int  b2v_set_qp(void* h, int32_t qp);                    /* CQP mode (restart-free set_crf) */
int  b2v_set_gop(void* h, int32_t frames);               /* b2v_settings.gop, live (the Python side converts keyframe_distance
                                                            SECONDS, settings.py:163, with the current fps) */
int  b2v_set_resolution(void* h, int32_t src_w, int32_t src_h, int32_t dst_w, int32_t dst_h);
int  b2v_request_idr(void* h);
int  b2v_set_max_picture_bytes(void* h, int32_t bytes);  /* B2V_FLAG_SIZE_CAP: the cap of every P picture from the next submit on
                                                            (0 = none, the default).  B2V_ESTATE without the flag, B2V_EINVAL
                                                            for a negative value. */

/* ---- quality of the record being delivered (B2V_FLAG_QUALITY) --------------
 * Valid only inside this session's frame callback, on its output thread: fills *out with the measurement of the record the
 * callback is delivering (the same lifetime rule as b2v_frame.data).  B2V_ESTATE outside a callback of this session or on a
 * session created without B2V_FLAG_QUALITY; B2V_EINVAL for a null handle or out. */
int  b2v_frame_quality(void* h, b2v_quality* out);

/* ---- introspection / test hooks ------------------------------------------- */
int  b2v_get_stats(void* h, b2v_stats* out);
int  b2v_reset_stats(void* h);
int  b2v_coded_size(void* h, int32_t* coded_w, int32_t* coded_h);
/* synchronous fused CSC(+scale) of one host BGRA frame to host NV12 (dst_w*dst_h*3/2 bytes) */
int  b2v_csc_nv12(void* h, const void* bgra_host, int32_t stride_bytes, void* nv12_host);
/* B2V_FLAG_DAMAGE's map of rectangles (source pixels, clipped to src_w x src_h) to the 16 x 16 tiles of a dst_w x dst_h output:
 * map[ty * ceil(dst_w / 16) + tx] = 1 when tile (tx, ty) must be converted again, else 0.  At 1:1 a tile is dirty when it meets a
 * rectangle; when scaling, when the source footprint of its bilinear taps meets one.  Padding rows and columns of the coded
 * picture lie in the tile of the last visible row or column.  Returns the count of dirty tiles, or B2V_EINVAL (sizes as
 * b2v_create takes them, rectangles as the damage submits take them, null map).  Host code, no CUDA call; the submits use it. */
int  b2v_damage_tiles(int32_t src_w, int32_t src_h, int32_t dst_w, int32_t dst_h, const b2v_rect* rects, int32_t n_rects, uint8_t* map);
/* the same of one device tensor, read in place after the work enqueued on `cuda_stream` (checked as b2v_submit_tensor checks it) */
int  b2v_csc_nv12_tensor(void* h, const b2v_tensor* t, void* cuda_stream, void* nv12_host);
/* reconstruction of the last encoded frame: NV12, coded_w*coded_h*3/2 bytes */
int  b2v_get_recon(void* h, void* nv12_host);
/* repeat the CSC kernel `iters` times over resident frames and return mean ms per launch
 * (CUDA events on the launching stream); used by bench.py for the roofline leg. */
int  b2v_bench_csc(void* h, int32_t n_resident, int32_t iters, float* ms_per_launch);
/* same, but `iters` launches back to back between ONE event pair (amortises the event/launch gap) */
int  b2v_bench_csc_burst(void* h, int32_t n_resident, int32_t iters, float* ms_per_launch);
/* device-side stopwatch on the encode stream: start = after everything submitted so far has drained;
 * stop = after every frame submitted since has been delivered.  bench.py times its K steps with it. */
int  b2v_timer_start(void* h);
int  b2v_timer_stop(void* h, float* ms);
const char* b2v_last_error(void);

/* ---- RTP H.264 payloader (SURVEY.md §8f row 1): replaces H264Encoder.pack -> _split_bitstream / _packetize
 *      (src/selkies/webrtc/codecs/h264.py:238-279, 331-335).  Splits the Annex-B access unit and writes the RTP
 *      payloads (single NAL, STAP-A, FU-A; RFC 6184 packetization-mode 1) back to back into `out`; lens[i] is the
 *      size of payload i.  Byte-identical to the reference (tests/golden/rtp_h264_golden.json).  Host code, no GPU.
 *      Returns B2V_ENOMEM when out/lens are too small (out_cap >= au_size + au_size/600 + 64 always suffices). */
int  b2v_rtp_h264_packetize(const uint8_t* au, int32_t au_size, int32_t packet_max, uint8_t* out, int32_t out_cap,
                            int32_t* lens, int32_t max_packets, int32_t* n_packets);

#ifdef __cplusplus
}
#endif
#endif /* B2VIDEO_H_ */
