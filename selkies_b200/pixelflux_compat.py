"""pixelflux-compatible module surface: `CaptureSettings`, `ScreenCapture`, `StripeCallback`.

The reference imports exactly these three names from the out-of-tree `pixelflux` wheel
(src/selkies/media_pipeline.py:28, src/selkies/selkies.py:90) and drives them as documented in
SURVEY.md §8b.  This module keeps that contract — same names, same attribute/method set, same
callback shape, same threading — on top of libb2video (CUDA, no CPU fallback):

    cs = CaptureSettings(); cs.capture_width = ...            # media_pipeline.py:251-273
    cap = ScreenCapture()
    cap.start_capture(cs, callback)                           # media_pipeline.py:299-300; selkies.py:3175
    cap.update_framerate(60.0); cap.update_video_bitrate(8000); cap.request_idr_frame()   # :236 :195 :244
    cap.stop_capture()                                        # :313 (blocking)

callback(result_ptr, user_data): `result_ptr.contents` has `.data`, `.size`, `.frame_id`;
`bytes(result.data[10:result.size])` (media_pipeline.py:286) and `bytes(result.data[:result.size])`
(selkies.py:3116) both work; `data` is only valid during the callback; the callback fires on the
library's native output thread.

What differs, by construction: the reference's module also grabs the X11 framebuffer.  Screen capture is
outside this tier (SURVEY.md §8b), so frames come from a pluggable `FrameSource` (default: a synthetic
desktop generator); a real grabber only has to fill the pinned ring slot it is handed.
"""
from __future__ import annotations

import ctypes as C
import threading
import time
from types import SimpleNamespace
from typing import Callable, Optional

import numpy as np

from . import _native as N
from .session import Session


class CaptureSettings:
    """Attribute bag with pixelflux's field names (SURVEY.md §8b).  Unknown attributes are accepted."""

    def __init__(self):
        self.capture_width = 1920
        self.capture_height = 1080
        self.capture_x = 0
        self.capture_y = 0
        self.target_fps = 60.0
        self.capture_cursor = False
        self.output_mode = 1                     # 0 = JPEG stripes (unsupported here), 1 = H.264
        self.auto_adjust_screen_capture_size = False
        self.h264_streaming_mode = False
        self.h264_fullframe = True
        self.h264_fullcolor = False
        self.h264_crf = 25                       # settings.py:48
        self.h264_paintover_crf = 18
        self.h264_paintover_burst_frames = 5
        self.h264_cbr_mode = False
        self.h264_bitrate_kbps = 8000            # settings.py:49 (8 Mbps)
        self.vaapi_render_node_index = -1
        self.use_cpu = False
        self.jpeg_quality = 60
        self.paint_over_jpeg_quality = 90
        self.use_paint_over_quality = False
        self.paint_over_trigger_frames = 15
        self.damage_block_threshold = 10
        self.damage_block_duration = 20
        self.scale = 1.0
        self.debug_logging = False
        self.watermark_path = b""
        self.watermark_location_enum = 0
        # additions of this implementation (ignored by the reference, which never sets them)
        self.gpu_id = 0                          # settings.py:162 exists but is never forwarded
        self.keyframe_distance = -1              # settings.py:163: SECONDS between key frames; <= 0 = only on request
        self.slice_rows = 0
        self.h264_stripe_rows = 0                # striped mode (h264_fullframe False): macroblock rows per stripe; 0 = about 8 stripes
        self.output_width = 0                    # != capture size => fused bilinear scale
        self.output_height = 0


class StripeCallback:
    """`StripeCallback(fn)` wrapper (selkies.py:3175); a bare callable is accepted too (media_pipeline.py:300)."""

    def __init__(self, fn: Callable):
        if not callable(fn):
            raise TypeError("StripeCallback needs a callable")
        self.fn = fn

    def __call__(self, result_ptr, user_data):
        return self.fn(result_ptr, user_data)


class _Result:
    __slots__ = ("data", "size", "frame_id", "is_key", "qp", "pts90k")


class _ResultPtr:
    """Stands in for `POINTER(StripeEncodeResult)`: truthy, `.contents` gives the result."""
    __slots__ = ("contents",)

    def __init__(self, r):
        self.contents = r

    def __bool__(self):
        return True


class FrameSource:
    """Producer of BGRA frames.  `fill(view, index)` writes frame `index` into a (H,W,4) uint8 view of a pinned
    ring slot; return False to end the stream."""

    def configure(self, width: int, height: int) -> None:
        self.width, self.height = width, height

    def fill(self, view: np.ndarray, index: int) -> bool:   # pragma: no cover - interface
        raise NotImplementedError


class SyntheticDesktopSource(FrameSource):
    """Flat regions, text-like 1-px patterns and a region scrolling 8 px/frame (SURVEY.md §8d S3)."""

    def __init__(self, seed: int = 1, distinct: int = 16):
        self.seed, self.distinct, self._cache = seed, distinct, None

    def configure(self, width, height):
        super().configure(width, height)
        self._cache = None

    def _frames(self):
        if self._cache is None:
            rng = np.random.default_rng(self.seed)
            w, h = self.width, self.height
            base = np.empty((h, w, 4), np.uint8)
            base[..., :3] = (240, 240, 240)
            base[..., 3] = 255
            base[: max(1, h // 12), :, :3] = (60, 40, 30)
            base[:, : max(1, w // 6), :3] = (200, 210, 220)
            th = h * 2 + 8 * self.distinct
            tw = w - w // 6
            glyph = rng.integers(0, 2, ((th + 1) // 2, (tw + 1) // 2), dtype=np.uint8).repeat(2, 0).repeat(2, 1)[:th, :tw]
            line = ((np.arange(th) // 8) % 3 != 2)[:, None]
            txt = np.where((glyph > 0) & line, 20, 240).astype(np.uint8)
            self._cache = (base, txt)
        return self._cache

    def fill(self, view, index):
        base, txt = self._frames()
        h, w = self.height, self.width
        y0 = max(1, h // 12)
        view[...] = base
        off = 8 * (index % self.distinct)
        region = txt[off: off + (h - y0), :]
        view[y0:, w // 6: w // 6 + region.shape[1], 0] = region
        view[y0:, w // 6: w // 6 + region.shape[1], 1] = region
        view[y0:, w // 6: w // 6 + region.shape[1], 2] = region
        return True


class ArraySource(FrameSource):
    """Cycles through pre-built frames (tests, benchmarks)."""

    def __init__(self, frames, loop: bool = True):
        self.frames, self.loop = list(frames), loop

    def fill(self, view, index):
        if index >= len(self.frames) and not self.loop:
            return False
        f = self.frames[index % len(self.frames)]
        if f.shape != view.shape:        # the display was resized: nearest-neighbour resample of the canned frame
            ys = (np.arange(view.shape[0]) * f.shape[0]) // view.shape[0]
            xs = (np.arange(view.shape[1]) * f.shape[1]) // view.shape[1]
            f = f[ys][:, xs]
        view[...] = f
        return True


class ScreenCapture:
    """One capture+encode instance (the reference keeps one per display, selkies.py:3178-3181)."""

    def __init__(self, frame_source: Optional[FrameSource] = None):
        self._source = frame_source
        self._session: Optional[Session] = None
        self._user_cb = None
        self._thread = None
        self._stop = threading.Event()
        self._lock = threading.RLock()           # control calls arrive on arbitrary executor threads
        self._resize_lock = threading.Lock()     # capture loop (acquire..submit) vs update_resolution; never held with _lock by the loop
        self._kf_seconds = -1.0
        self._fps = 60.0
        self._cursor_cb = None
        self.frames_emitted = 0

    # -- lifecycle ----------------------------------------------------------------------------------
    def start_capture(self, settings: CaptureSettings, callback) -> None:
        with self._lock:
            if self._session is not None:
                raise RuntimeError("capture already running")
            jpeg = int(getattr(settings, "output_mode", 1)) == 0        # the reference's "jpeg" encoder (selkies.py:3209-3212)
            if not callable(callback):
                raise TypeError("callback must be callable or a StripeCallback")
            if not jpeg and bool(getattr(settings, "h264_fullcolor", False)):
                # The client picks a SUPERSET decoder configuration for this switch (avc1.F400xx, High 4:4:4 Predictive;
                # selkies-ws-core.js:475-496), under which a Constrained-Baseline 4:2:0 stream decodes as well: the stream stays
                # 4:2:0 (chroma at half resolution) instead of the capture failing.
                import warnings
                warnings.warn("h264_fullcolor: this pipeline encodes 4:2:0 (Constrained Baseline); the stream decodes under the 4:4:4 decoder "
                              "configuration the client selects, with chroma at half resolution", RuntimeWarning, stacklevel=2)
            w, h = int(settings.capture_width), int(settings.capture_height)
            w -= w & 1
            h -= h & 1                                # the reference forces even sizes (webrtc_mode.py:397-402)
            s = SimpleNamespace(paintover_trigger_frames=0, paintover_crf=0, paintover_burst_frames=0)      # Session keyword arguments; paint-over off
            s.dst_width, s.dst_height = int(getattr(settings, "output_width", 0) or 0), int(getattr(settings, "output_height", 0) or 0)
            s.fps = float(settings.target_fps) if float(settings.target_fps) > 0 else 60.0
            s.device = int(getattr(settings, "gpu_id", 0) or 0)
            s.rc_mode = N.B2V_RC_CBR if bool(settings.h264_cbr_mode) else N.B2V_RC_CQP
            s.bitrate_kbps = int(settings.h264_bitrate_kbps)
            s.crf = int(settings.h264_crf)
            self._kf_seconds = float(getattr(settings, "keyframe_distance", -1) or -1)
            s.gop = self._gop_frames(self._kf_seconds, s.fps)
            s.slice_rows = int(getattr(settings, "slice_rows", 0) or 0)
            s.header_mode = N.B2V_HDR_PIXELFLUX       # callers strip / keep the 10-byte header themselves
            s.ring_slots = 4
            s.flags = 0
            if bool(getattr(settings, "use_paint_over_quality", False)):
                # selkies.py:3217, 3226-3229: after paint_over_trigger_frames static pictures, h264_paintover_burst_frames pictures
                # are coded at h264_paintover_crf (in CBR mode only when that is finer than the rate controller's QP)
                s.paintover_trigger_frames = int(getattr(settings, "paint_over_trigger_frames", 15) or 0)
                s.paintover_crf = int(getattr(settings, "h264_paintover_crf", 18))
                s.paintover_burst_frames = max(1, int(getattr(settings, "h264_paintover_burst_frames", 1) or 1))
            if not bool(getattr(settings, "h264_fullframe", True)):
                # "x264enc-striped" (selkies.py:3219): independent H.264 stripes, unchanged stripes are not sent
                sl = max(1, s.slice_rows)
                rows = int(getattr(settings, "h264_stripe_rows", 0) or 0)
                if rows <= 0:
                    mbh = ((s.dst_height or h) + 15) // 16
                    rows = -(-mbh // 8)
                s.stripe_rows = -(-rows // sl) * sl
            if jpeg:
                # JPEG stripes: each changed stripe is one JFIF file behind frame_id | y_start; unchanged stripes are not sent, a
                # stripe static for paint_over_trigger_frames pictures is sent once more at paint_over_jpeg_quality
                s.flags |= N.B2V_FLAG_JPEG
                s.rc_mode = N.B2V_RC_CQP
                s.crf = int(getattr(settings, "jpeg_quality", 60))
                s.paintover_crf = int(getattr(settings, "paint_over_jpeg_quality", 90))
                s.paintover_trigger_frames = int(getattr(settings, "paint_over_trigger_frames", 15) or 0) if bool(getattr(settings, "use_paint_over_quality", False)) else 0
                s.stripe_rows = int(getattr(settings, "h264_stripe_rows", 0) or 0)
            self._user_cb = callback
            # raises if the CUDA library is missing: no CPU fallback
            self._session = Session(w, h, collect=False, on_frame=self._on_frame, **vars(s))
            self._fps = s.fps
            if self._source is None:
                self._source = SyntheticDesktopSource()
            self._source.configure(w, h)
            self._stop.clear()
            self._thread = threading.Thread(target=self._capture_loop, name="b2v-capture", daemon=True)
            self._thread.start()

    def stop_capture(self) -> None:
        """Blocking: joins the capture thread and drains the encoder (media_pipeline.py:313)."""
        with self._lock:
            t = self._thread
            if self._session is None:
                return
            self._stop.set()
        if t is not None and t is not threading.current_thread():
            t.join()
        with self._lock:
            if self._session is not None:
                self._session.close()
                self._session = None
            self._thread = None

    @staticmethod
    def _gop_frames(seconds: float, fps: float) -> int:
        """keyframe_distance is in SECONDS (settings.py:163); the session's gop is in frames."""
        return -1 if seconds <= 0 else max(1, int(round(seconds * fps)))

    # -- live control ----------------------------------------------------------------------------------
    def update_framerate(self, fps: float) -> None:
        with self._lock:
            if self._session is None:
                return
            self._session.set_framerate(fps)
            self._fps = float(fps)
            if self._kf_seconds > 0:               # the key-frame interval is a time: keep it across the rate change
                self._session.set_gop(self._gop_frames(self._kf_seconds, self._fps))

    def update_video_bitrate(self, kbps: int) -> None:
        with self._lock:
            if self._session is None:
                return
            self._session.set_bitrate_kbps(kbps)

    def request_idr_frame(self) -> None:
        with self._lock:
            if self._session is None:
                return
            self._session.request_idr()

    def update_resolution(self, width: int, height: int) -> None:
        """Follow a display resize (what auto_adjust_screen_capture_size does in the reference)."""
        with self._resize_lock:                  # the capture loop holds no ring slot while we are in here
            with self._lock:
                if self._session is None:
                    return
                width -= width & 1
                height -= height & 1
                self._session.set_resolution(width, height)
                self._source.configure(width, height)

    def set_cursor_callback(self, fn) -> None:       # selkies.py:3166-3167 (guarded by hasattr)
        self._cursor_cb = fn

    # -- internals ----------------------------------------------------------------------------------------
    def _capture_loop(self):
        index = 0
        next_t = time.perf_counter()
        while not self._stop.is_set():
            # The control lock is held only for the snapshot: acquire (blocks while the ring is full), fill (tens of ms at 4K) and
            # submit run outside it, so request_idr_frame / update_* never queue behind a frame and a callback that calls them
            # while the ring is full cannot deadlock.  The session stays open: stop_capture joins this thread before closing it.
            with self._lock:
                session, fps = self._session, self._fps
            if session is None:
                break
            with self._resize_lock:
                try:
                    slot, view = session.acquire()
                except N.B2VError:
                    break                         # the session is stopping
                if not self._source.fill(view, index):
                    session.release_slot(slot)    # end of the source: nothing to encode
                    break
                session.submit_slot(slot, time.monotonic_ns())
            index += 1
            next_t += 1.0 / max(1e-3, fps)
            delay = next_t - time.perf_counter()
            if delay > 0:
                self._stop.wait(delay)
            else:
                next_t = time.perf_counter()      # fell behind: do not burst

    def _on_frame(self, fptr):
        f = fptr.contents
        r = _Result()
        # zero-copy view of the native buffer, valid for the duration of the callback only
        r.data = memoryview((C.c_ubyte * f.size).from_address(C.addressof(f.data.contents))).cast("B")
        r.size = f.size
        r.frame_id = f.frame_id
        r.is_key = f.is_key
        r.qp = f.qp
        r.pts90k = f.pts90k
        self.frames_emitted += 1
        try:
            self._user_cb(_ResultPtr(r), None)
        finally:
            try:
                r.data.release()
            except BufferError:      # the callee kept a buffer export alive; the bytes are stale after return
                pass
