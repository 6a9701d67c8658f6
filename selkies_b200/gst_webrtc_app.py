"""`GSTWebRTCApp`-named façade: the legacy selkies-gstreamer video surface BASELINE.json names
(build_video_pipeline / set_framerate / set_resolution / set_video_bitrate), kept so the pipeline drops
in as the video branch feeding the existing payloader -> webrtcbin sink.

That class is not in the reference snapshot (SURVEY.md §0: only a vestigial kwarg at
src/selkies/webrtc_mode.py:163); its four methods map onto what the snapshot does have:
  build_video_pipeline -> MediaPipelinePixel.generate_capture_settings + start_screen_capture (media_pipeline.py:251-306)
  set_framerate        -> MediaPipelinePixel.set_framerate  (media_pipeline.py:223-237)
  set_video_bitrate    -> MediaPipelinePixel.set_video_bitrate (media_pipeline.py:183-201; legacy unit was kbps)
  set_resolution       -> WebRTCApp.on_resize_handler (webrtc_mode.py:383-426)
The façade is synchronous (the legacy class was driven from GLib callbacks, not asyncio).
"""
from __future__ import annotations

import logging
from typing import Callable, Optional

from .pixelflux_compat import CaptureSettings, FrameSource, ScreenCapture

logger = logging.getLogger("gstwebrtc_app_b200")


class GSTWebRTCAppError(Exception):
    pass


class GSTWebRTCApp:
    def __init__(self, encoder: str = "x264enc", framerate: int = 60, video_bitrate: int = 8000, width: int = 1920,
                 height: int = 1080, gpu_id: int = 0, keyframe_distance: float = -1, cbr: bool = True, crf: int = 25,
                 frame_source: Optional[FrameSource] = None):
        self.encoder = encoder
        self.framerate = framerate
        self.video_bitrate = video_bitrate          # kbps, as in the legacy class
        self.width, self.height = width, height
        self.gpu_id = gpu_id
        self.keyframe_distance = keyframe_distance
        self.cbr, self.crf = cbr, crf
        self.frame_source = frame_source
        self.capture: Optional[ScreenCapture] = None
        # sink hook: (annexb_bytes, pts_90khz, is_key) -> None; default drops (wire it to rtph264pay/RTCApp.consume_data)
        self.on_video_sample: Callable[[bytes, int, bool], None] = lambda data, pts, key: None
        self.frames = 0

    def _callback(self, result_ptr, _):
        if not result_ptr:
            return
        r = result_ptr.contents
        if r.size <= 10:
            return
        pts = r.frame_id * (90000 // max(1, int(self.framerate)))
        self.frames += 1
        self.on_video_sample(bytes(r.data[10:r.size]), pts, bool(r.is_key))

    def build_video_pipeline(self) -> None:
        if self.capture is not None:
            raise GSTWebRTCAppError("video pipeline already built")
        if self.encoder not in ("x264enc", "nvh264enc", "b200h264enc"):
            raise GSTWebRTCAppError(f"unsupported encoder {self.encoder!r} for the CUDA video branch")
        cs = CaptureSettings()
        cs.capture_width, cs.capture_height = self.width, self.height
        cs.target_fps = float(self.framerate)
        cs.output_mode = 1
        cs.h264_streaming_mode = True
        cs.h264_fullframe = True
        cs.h264_cbr_mode = self.cbr
        cs.h264_crf = self.crf
        cs.h264_bitrate_kbps = int(self.video_bitrate)
        cs.gpu_id = self.gpu_id
        cs.keyframe_distance = self.keyframe_distance
        cap = ScreenCapture(self.frame_source)
        cap.start_capture(cs, self._callback)
        self.capture = cap

    def stop_pipeline(self) -> None:
        if self.capture is not None:
            self.capture.stop_capture()
            self.capture = None

    def _need(self) -> ScreenCapture:
        if self.capture is None:
            raise GSTWebRTCAppError("video pipeline not built")
        return self.capture

    def set_framerate(self, framerate: int) -> None:
        if framerate <= 0:
            raise GSTWebRTCAppError("framerate must be positive")
        self._need().update_framerate(float(framerate))
        self.framerate = framerate

    def set_video_bitrate(self, bitrate: int) -> None:
        """:bitrate: kbps (legacy GSTWebRTCApp unit)."""
        if bitrate <= 0:
            raise GSTWebRTCAppError("bitrate must be positive")
        self._need().update_video_bitrate(int(bitrate))
        self.video_bitrate = bitrate

    def set_resolution(self, width: int, height: int) -> None:
        width -= width & 1
        height -= height & 1
        if width < 16 or height < 16 or width > 7680 or height > 4320:
            raise GSTWebRTCAppError(f"resolution {width}x{height} out of range")
        self._need().update_resolution(width, height)
        self.width, self.height = width, height

    def send_idr(self) -> None:                       # PLI -> IDR (rtc.py:601-603)
        self._need().request_idr_frame()
