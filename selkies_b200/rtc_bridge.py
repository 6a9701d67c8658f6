"""Hand-off from the encoder callback to the RTP sender (SURVEY.md §8 rows a11, f3).

Reference: `RTCApp.consume_data` wraps every access unit in `av.Packet(bytes(buf))` with `time_base = 1/90000`, `pts = dts`
and puts it into `PipelineBridge`, a depth-1 drop-oldest `asyncio.Queue` (src/selkies/rtc.py:102-118, 408-421); the sender later
calls `encoder.pack(packet)` on it (rtcrtpsender.py:362).  `av` is not needed for any of that — the packet is only a bag for
bytes + pts — so `VideoSample` carries the same attributes, `consume_data` makes ONE copy of the callback's view (the reference
makes two: `bytes(ptr[10:size])` then `bytes(buf)`), and `pack()` returns the RTP payloads from the native payloader.
"""
from __future__ import annotations

import asyncio
from fractions import Fraction
from typing import Any, Optional

from .h264_nal import is_droppable

RTP_VIDEO_CLOCK_RATE = 90000


class PipelineBridge:
    """Newest-sample-wins mailbox between the encoder callback and the RTP sender: same contract as the reference's bridge
    (rtc.py:102-118: a lagging consumer sees the newest sample only; `get_data` waits for one).  Everything happens on the
    event loop and `set_data` never yields between the drop and the put, so no lock is involved.

    A reference sample is never dropped while a droppable one can go (B2V_FLAG_DROPPABLE: nothing predicts from a droppable
    sample, so the stream stays decodable without it): a waiting droppable sample is replaced; a new droppable sample arriving
    while a reference sample waits is dropped itself; of two reference samples the older is dropped, as without the flag, and
    also counted in `dropped_reference` (the decoder predicts from a picture it never got until the next IDR).  A sample
    without a `droppable` attribute counts as a reference sample."""

    def __init__(self):
        self._slot: asyncio.Queue = asyncio.Queue(maxsize=1)
        self.dropped = 0
        self.dropped_reference = 0

    async def set_data(self, data: Any):
        while self._slot.full():
            old = self._slot.get_nowait()
            self.dropped += 1
            if getattr(old, "droppable", False):
                continue
            if getattr(data, "droppable", False):
                self._slot.put_nowait(old)             # the waiting reference sample stays, the new droppable one goes
                return
            self.dropped_reference += 1
        self._slot.put_nowait(data)

    async def get_data(self):
        return await self._slot.get()


class VideoSample:
    """What the sender needs of `av.Packet`: bytes(sample), .pts, .dts, .time_base, .is_keyframe; and .droppable, read from the
    access unit: a non-reference picture (B2V_FLAG_DROPPABLE) that PipelineBridge sheds first."""
    __slots__ = ("data", "pts", "dts", "time_base", "is_keyframe", "droppable")

    def __init__(self, data: bytes, pts: Optional[int], is_keyframe: bool = False):
        self.data, self.pts, self.dts = data, pts, pts
        self.time_base = Fraction(1, RTP_VIDEO_CLOCK_RATE)
        self.is_keyframe = is_keyframe
        self.droppable = is_droppable(data)

    def __bytes__(self):
        return self.data

    def __len__(self):
        return len(self.data)


class VideoBridge:
    """`consume_data(buf, pts, "video")` + `pack(sample)` for the video branch of RTCApp."""

    def __init__(self, payloader=None):
        self.video_pipeline_bridge = PipelineBridge()
        self._payloader = payloader            # created lazily: needs libb2video

    async def consume_data(self, buf, pts, kind: str = "video", is_keyframe: bool = False):
        if kind != "video" or not buf:
            return
        data = buf if isinstance(buf, bytes) else bytes(buf)       # a memoryview of the pinned slot is copied once, here
        await self.video_pipeline_bridge.set_data(VideoSample(data, pts, is_keyframe))

    def pack(self, sample: VideoSample):
        """`H264Encoder.pack(packet)` (webrtc/codecs/h264.py:331-335): (payloads, 90 kHz timestamp)."""
        if self._payloader is None:
            from .rtp_h264 import H264Payloader
            self._payloader = H264Payloader()
        den = sample.time_base.denominator // max(1, sample.time_base.numerator)
        return self._payloader.pack(sample.data, sample.pts or 0, den)
