"""Thin object wrapper over one libb2video session handle (include/b2video.h).

One Session = one encoder instance on one GPU: what one `pixelflux.ScreenCapture`
is in the reference (one per display, selkies.py:3178-3181).  Used by
pixelflux_compat.ScreenCapture, bench.py and the tests.
"""
from __future__ import annotations

import ctypes as C
import threading
from typing import Callable, Optional

import numpy as np

from . import _native as N


class EncodedFrame:
    __slots__ = ("data", "frame_id", "is_key", "qp", "pts90k", "capture_ns", "y_start", "height")

    def __init__(self, data: bytes, frame_id: int, is_key: bool, qp: int, pts90k: int, capture_ns: int, y_start: int = 0, height: int = 0):
        self.data = data
        self.frame_id = frame_id
        self.is_key = is_key
        self.qp = qp
        self.pts90k = pts90k
        self.capture_ns = capture_ns
        self.y_start, self.height = y_start, height


class Session:
    def __init__(self, width: int, height: int, *, dst_width: int = 0, dst_height: int = 0, fps: float = 60.0,
                 device: int = 0, rc_mode: int = N.B2V_RC_CBR, bitrate_kbps: int = 8000, crf: int = 26,
                 gop: int = -1, slice_rows: int = 0, paintover_trigger_frames: int = 0, paintover_crf: int = 18, paintover_burst_frames: int = 1, idr_slice_mbs: int = 0, stripe_rows: int = 0, header_mode: int = N.B2V_HDR_NONE, ring_slots: int = 4,
                 flags: int = 0, on_frame: Optional[Callable[[C.POINTER(N.B2VFrame)], None]] = None,
                 collect: bool = True):
        self._lib = N.lib()
        self.width, self.height = width, height
        self.dst_width, self.dst_height = dst_width or width, dst_height or height
        self.frames: list[EncodedFrame] = []
        self._collect = collect
        self._on_frame = on_frame
        self._lock = threading.Lock()
        s = N.B2VSettings()
        s.src_w, s.src_h, s.dst_w, s.dst_h = width, height, dst_width, dst_height
        s.fps, s.device, s.rc_mode, s.bitrate_kbps, s.crf = float(fps), device, rc_mode, bitrate_kbps, crf
        s.gop, s.slice_rows, s.header_mode, s.ring_slots, s.flags = gop, slice_rows, header_mode, ring_slots, flags
        s.paintover_trigger_frames, s.paintover_crf, s.stripe_rows = paintover_trigger_frames, paintover_crf, stripe_rows
        s.paintover_burst_frames, s.idr_slice_mbs = paintover_burst_frames, idr_slice_mbs
        # keep alive for the lifetime of the handle.  With nothing to deliver to Python the library gets no callback at all: a
        # ctypes callback takes the GIL on the output thread for every picture, which costs the submitting thread its pace.
        self._cb = N.FRAME_CB(self._callback) if (on_frame is not None or collect) else N.FRAME_CB()
        h = C.c_void_p()
        N.check(self._lib.b2v_create(C.byref(s), self._cb, None, C.byref(h)))
        self._h = h

    # -- native callback (fires on the library's output thread) ------------------------------
    def _callback(self, fptr, _user):
        if self._on_frame is not None:
            self._on_frame(fptr)
        if self._collect:
            f = fptr.contents
            rec = EncodedFrame(C.string_at(f.data, f.size), f.frame_id, bool(f.is_key), f.qp, f.pts90k, f.capture_ns, f.y_start, f.height)
            with self._lock:
                self.frames.append(rec)

    # -- ingest ---------------------------------------------------------------------------------
    def submit(self, bgra: np.ndarray, capture_ns: int = 0) -> None:
        """Copy one (H,W,4) uint8 BGRA frame into the next pinned ring slot and enqueue it."""
        assert bgra.dtype == np.uint8 and bgra.shape == (self.height, self.width, 4), bgra.shape
        slot = C.c_int32(-1)
        p = self._lib.b2v_ring_acquire(self._h, C.byref(slot))
        if not p:
            N.check(N.B2V_ESTATE)
        C.memmove(p, np.ascontiguousarray(bgra).ctypes.data, self.width * self.height * 4)
        N.check(self._lib.b2v_ring_submit(self._h, slot.value, self.width * 4, capture_ns))

    def acquire(self):
        """Zero-copy ingest: returns (slot, numpy view of the pinned slot) to fill in place."""
        slot = C.c_int32(-1)
        p = self._lib.b2v_ring_acquire(self._h, C.byref(slot))
        if not p:
            N.check(N.B2V_ESTATE)
        buf = (C.c_ubyte * (self.width * self.height * 4)).from_address(p)
        return slot.value, np.frombuffer(buf, np.uint8).reshape(self.height, self.width, 4)

    def release_slot(self, slot: int) -> None:
        """Give the most recently acquired slot back without encoding it."""
        N.check(self._lib.b2v_ring_release(self._h, slot))

    def submit_slot(self, slot: int, capture_ns: int = 0) -> None:
        N.check(self._lib.b2v_ring_submit(self._h, slot, self.width * 4, capture_ns))

    def resident_upload(self, index: int, bgra: np.ndarray) -> None:
        bgra = np.ascontiguousarray(bgra)
        N.check(self._lib.b2v_resident_upload(self._h, index, bgra.ctypes.data, self.width * 4))

    def submit_resident(self, index: int, capture_ns: int = 0) -> None:
        N.check(self._lib.b2v_submit_resident(self._h, index, capture_ns))

    def flush(self) -> None:
        N.check(self._lib.b2v_flush(self._h))

    # -- control ----------------------------------------------------------------------------------
    def set_framerate(self, fps: float) -> None:
        N.check(self._lib.b2v_set_framerate(self._h, float(fps)))

    def set_bitrate_kbps(self, kbps: int) -> None:
        N.check(self._lib.b2v_set_bitrate_kbps(self._h, int(kbps)))

    def set_qp(self, qp: int) -> None:
        N.check(self._lib.b2v_set_qp(self._h, int(qp)))

    def set_resolution(self, width: int, height: int, dst_width: int = 0, dst_height: int = 0) -> None:
        N.check(self._lib.b2v_set_resolution(self._h, width, height, dst_width, dst_height))
        self.width, self.height = width, height
        self.dst_width, self.dst_height = dst_width or width, dst_height or height

    def set_gop(self, frames: int) -> None:
        """Key-frame distance in pictures from the next submit on (<= 0: key frames only on request)."""
        N.check(self._lib.b2v_set_gop(self._h, int(frames)))

    def request_idr(self) -> None:
        N.check(self._lib.b2v_request_idr(self._h))

    # -- introspection ----------------------------------------------------------------------------
    def coded_size(self):
        w, h = C.c_int32(), C.c_int32()
        N.check(self._lib.b2v_coded_size(self._h, C.byref(w), C.byref(h)))
        return w.value, h.value

    def stats(self) -> dict:
        st = N.B2VStats()
        N.check(self._lib.b2v_get_stats(self._h, C.byref(st)))
        return st.as_dict()

    def reset_stats(self) -> None:
        N.check(self._lib.b2v_reset_stats(self._h))

    def csc_nv12(self, bgra: np.ndarray):
        """Synchronous fused CSC(+scale): returns (Y (dh,dw), UV (dh/2,dw)) uint8."""
        bgra = np.ascontiguousarray(bgra)
        assert bgra.shape == (self.height, self.width, 4)
        dw, dh = self.dst_width, self.dst_height
        out = np.empty(dw * dh * 3 // 2, np.uint8)
        N.check(self._lib.b2v_csc_nv12(self._h, bgra.ctypes.data, self.width * 4, out.ctypes.data))
        return out[: dw * dh].reshape(dh, dw), out[dw * dh:].reshape(dh // 2, dw)

    def recon(self):
        cw, ch = self.coded_size()
        out = np.empty(cw * ch * 3 // 2, np.uint8)
        N.check(self._lib.b2v_get_recon(self._h, out.ctypes.data))
        return out[: cw * ch].reshape(ch, cw), out[cw * ch:].reshape(ch // 2, cw)

    def bench_csc(self, n_resident: int, iters: int) -> float:
        ms = C.c_float()
        N.check(self._lib.b2v_bench_csc(self._h, n_resident, iters, C.byref(ms)))
        return float(ms.value)

    def bench_csc_burst(self, n_resident: int, iters: int) -> float:
        ms = C.c_float()
        N.check(self._lib.b2v_bench_csc_burst(self._h, n_resident, iters, C.byref(ms)))
        return float(ms.value)

    def timer_start(self) -> None:
        N.check(self._lib.b2v_timer_start(self._h))

    def timer_stop(self) -> float:
        ms = C.c_float()
        N.check(self._lib.b2v_timer_stop(self._h, C.byref(ms)))
        return float(ms.value)

    def take_frames(self) -> list:
        with self._lock:
            out, self.frames = self.frames, []
        return out

    def close(self) -> None:
        if self._h:
            self._lib.b2v_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
