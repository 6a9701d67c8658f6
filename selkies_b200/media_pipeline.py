"""Video side of the selkies media-pipeline interface, backed by the CUDA encoder of this package.

The rest of selkies talks to an object with ten methods (the abstract class at src/selkies/media_pipeline.py:41-80) and two
callback attributes (`produce_data(buf, pts, kind)`, `send_data_channel_message(msg)`).  `MediaPipelineB200` offers that
object for the video path: constructor keywords, attribute names (`framerate`, `video_bitrate` in Mbit/s, `h264_crf`,
`rc_mode`, `width`, `height`, `capture_cursor`, `last_resize_success`, `capture_module`, `async_lock`) and the observable
rules of `MediaPipelinePixel` (media_pipeline.py:82-429) are kept:

* a setter does nothing while capture is not running, for an unchanged value, or for a value the mode does not use
  (bitrate in CRF mode, CRF in CBR mode, non-positive numbers);
* framerate, bitrate and key-frame requests reach the running encoder (`update_framerate`, `update_video_bitrate(kbps)`,
  `request_idr_frame`), on an executor thread; cursor visibility, rate-control mode and CRF re-create the capture;
* every encoded frame is handed to `produce_data` without its 10-byte stripe header, with `pts = frame_id * (90000 // fps)`.

Implementation notes: the parameters that need a re-created capture go through one `_respawn_with()` path, the live ones
through `_poke()`, so the guard rules live in one place each.  Audio (pcmflux) is outside this tier — `set_audio_bitrate`
is accepted and ignored.  `set_resolution()` is an addition (the reference writes `width/height` and relies on
`auto_adjust_screen_capture_size`, webrtc_mode.py:383-426).
"""
from __future__ import annotations

import asyncio
import logging
from abc import ABCMeta, abstractmethod
from enum import Enum
from typing import Any, Callable, Optional

from .pixelflux_compat import CaptureSettings, ScreenCapture

logger = logging.getLogger("media_pipeline_b200")
logger.setLevel(logging.INFO)

H264_ENCODER_NAMES = ("x264enc", "nvh264enc")      # names the reference's settings use for full-frame H.264
MIN_SIDE, MAX_W, MAX_H = 16, 7680, 4320            # selkies.py:281


class RateControlMode(str, Enum):
    CBR = "cbr"
    CRF = "crf"


class MediaPipelineError(Exception):
    pass


class MediaPipeline(metaclass=ABCMeta):
    """The ten entry points selkies calls on a media pipeline."""

    # lifecycle
    @abstractmethod
    def start_media_pipeline(self): ...

    @abstractmethod
    def stop_media_pipeline(self): ...

    @abstractmethod
    def is_media_pipeline_running(self) -> bool: ...

    # live controls
    @abstractmethod
    async def set_framerate(self, framerate: int): ...

    @abstractmethod
    async def set_video_bitrate(self, bitrate: int): ...

    @abstractmethod
    async def set_audio_bitrate(self, bitrate: int): ...

    @abstractmethod
    async def dynamic_idr_frame(self): ...

    # controls that re-create the capture
    @abstractmethod
    async def set_pointer_visible(self, visible: bool): ...

    @abstractmethod
    async def update_rate_control_mode(self, mode: RateControlMode): ...

    @abstractmethod
    async def set_crf(self, crf: int): ...


def _unwired(name: str) -> Callable[..., None]:
    def warn(*_a, **_k):
        logger.warning("%s is not wired to a consumer", name)
    return warn


class MediaPipelineB200(MediaPipeline):
    def __init__(self, async_event_loop: asyncio.AbstractEventLoop, encoder_rtc: str = "x264enc", framerate: int = 30,
                 video_bitrate: int = 8, audio_bitrate: int = 128000, width: int = 1920, height: int = 1080,
                 audio_channels: int = 2, audio_enabled: bool = False, audio_device_name="output.monitor",
                 crf: int = 23, rc_mode: RateControlMode = RateControlMode.CBR, gpu_id: int = 0, frame_source=None):
        self.async_event_loop = async_event_loop
        self.async_lock = asyncio.Lock()
        # what selkies reads back
        self.encoder_rtc, self.gpu_id = encoder_rtc, gpu_id
        self.width, self.height, self.framerate = width, height, framerate
        self.video_bitrate, self.h264_crf, self.rc_mode = video_bitrate, crf, rc_mode        # Mbit/s, QP, mode
        self.capture_cursor = False
        self.last_resize_success = True
        # audio parameters are only carried
        self.audio_bitrate, self.audio_channels = audio_bitrate, audio_channels
        self.audio_enabled, self.audio_device_name = audio_enabled, audio_device_name
        # consumers
        self.produce_data = _unwired("produce_data")
        self.send_data_channel_message = _unwired("send_data_channel_message")
        # capture state
        self.frame_source = frame_source
        self.capture_module: Optional[ScreenCapture] = None
        self._capturing = False
        self._started = False

    # ------------------------------------------------------------------------------------------ helpers
    def _live(self) -> Optional[ScreenCapture]:
        """The running capture object, or None when there is nothing to control."""
        return self.capture_module if self._capturing else None

    async def _off_loop(self, fn: Callable[..., Any], *args):
        return await self.async_event_loop.run_in_executor(None, fn, *args)

    async def _poke(self, method: str, *args) -> bool:
        """Call a live-control method of the capture object on an executor thread.  A capture module without the method is
        tolerated (the reference treats AttributeError as "feature unsupported")."""
        cap = self._live()
        if cap is None:
            return False
        fn = getattr(cap, method, None)
        if fn is None:
            logger.error("capture module has no %s()", method)
            return False
        try:
            await self._off_loop(fn, *args)
            return True
        except Exception as exc:
            logger.error("%s%r failed: %s", method, args, exc, exc_info=True)
            return False

    async def _respawn_with(self, attr: str, value) -> None:
        """Store a parameter that only takes effect at capture start, then stop and start the capture."""
        if self._live() is None or getattr(self, attr) == value:
            return
        setattr(self, attr, value)
        await self.restart_screen_capture()

    # ------------------------------------------------------------------------------------------ controls that respawn
    async def set_pointer_visible(self, visible: bool):
        await self._respawn_with("capture_cursor", visible)

    async def update_rate_control_mode(self, mode: RateControlMode):
        if mode not in (RateControlMode.CBR, RateControlMode.CRF):
            logger.error("unknown rate control mode %r", mode)
            return
        await self._respawn_with("rc_mode", mode)

    async def set_crf(self, new_crf: int):
        if self.rc_mode == RateControlMode.CRF:
            await self._respawn_with("h264_crf", new_crf)

    # ------------------------------------------------------------------------------------------ live controls
    async def set_video_bitrate(self, new_bitrate: int):
        """`new_bitrate` in Mbit/s (the unit of settings.py:49); the encoder takes kbit/s."""
        if self.rc_mode == RateControlMode.CRF or new_bitrate <= 0 or new_bitrate == self.video_bitrate:
            return
        if await self._poke("update_video_bitrate", int(new_bitrate) * 1000):
            self.video_bitrate = new_bitrate

    async def set_audio_bitrate(self, new_bitrate: int):
        return None

    async def set_framerate(self, framerate: int):
        async with self.async_lock:
            if framerate <= 0 or framerate == self.framerate or self._live() is None:
                return
            self.framerate = framerate               # the pts step of the callback follows
            await self._poke("update_framerate", float(framerate))

    async def dynamic_idr_frame(self):
        await self._poke("request_idr_frame")

    async def set_resolution(self, width: int, height: int):
        """Resize: even sizes only (the server rounds down, webrtc_mode.py:397-402); the encoder answers with new SPS/PPS + IDR."""
        width, height = width & ~1, height & ~1
        self.last_resize_success = MIN_SIDE <= width <= MAX_W and MIN_SIDE <= height <= MAX_H
        if not self.last_resize_success:
            return
        self.width, self.height = width, height
        await self._poke("update_resolution", width, height)

    # ------------------------------------------------------------------------------------------ capture life cycle
    def generate_capture_settings(self) -> CaptureSettings:
        cs = CaptureSettings()
        cs.capture_width, cs.capture_height, cs.capture_x, cs.capture_y = self.width, self.height, 0, 0
        cs.target_fps = float(self.framerate)
        cs.capture_cursor = self.capture_cursor
        cs.output_mode = 1                            # H.264
        cs.auto_adjust_screen_capture_size = True
        cs.gpu_id = self.gpu_id
        if self.encoder_rtc in H264_ENCODER_NAMES:
            cs.h264_streaming_mode = cs.h264_fullframe = True
            cs.h264_cbr_mode = self.rc_mode == RateControlMode.CBR
            cs.h264_crf = self.h264_crf
            cs.h264_bitrate_kbps = self.video_bitrate * 1000
            cs.vaapi_render_node_index = -1
            cs.use_cpu = self.encoder_rtc == "x264enc"      # carried for compatibility; the encode always runs on the GPU
        return cs

    def _on_encoded(self, result_ptr, _user) -> None:
        """Native output thread -> event loop.  The view is only valid during this call, so the payload is copied here, once."""
        if not result_ptr:
            return
        try:
            res = result_ptr.contents
            if res.size <= 0:
                return
            payload = bytes(res.data[10:res.size])
            pts = res.frame_id * (90000 // max(1, int(self.framerate)))
            asyncio.run_coroutine_threadsafe(self.produce_data(payload, pts, "video"), self.async_event_loop)
        except Exception as exc:                      # never let an exception travel back into the native thread
            logger.error("encoded-frame callback failed: %s", exc)

    async def start_screen_capture(self):
        if self._capturing:
            return
        cap = ScreenCapture(self.frame_source)
        try:
            await self._off_loop(cap.start_capture, self.generate_capture_settings(), self._on_encoded)
        except Exception as exc:
            logger.error("capture did not start: %s", exc, exc_info=True)
            self.capture_module, self._capturing = None, False
            return
        self.capture_module, self._capturing = cap, True

    async def stop_screen_capture(self):
        cap = self._live()
        if cap is None:
            return
        try:
            await self._off_loop(cap.stop_capture)
        except Exception as exc:
            logger.error("capture did not stop cleanly: %s", exc, exc_info=True)
        self.capture_module, self._capturing = None, False

    async def restart_screen_capture(self):
        if not self._capturing:
            return
        async with self.async_lock:
            await self.stop_screen_capture()
            await self.start_screen_capture()

    async def start_media_pipeline(self):
        async with self.async_lock:
            if not self._started:
                await self.start_screen_capture()
                self._started = self._capturing

    async def stop_media_pipeline(self):
        async with self.async_lock:
            if self._started:
                await self.stop_screen_capture()
                self._started = False

    def is_media_pipeline_running(self) -> bool:
        return self._started
