"""Scripted two-sided driver: one event list applied to a GPU `Session` and to `oracle.RefEncoder`, compared picture by picture.
Every H.264 parity test that drives a `Session` runs through it.

Events (plain tuples, built by the helpers below): picture(frame), set_bitrate(kbps), set_fps(fps), set_qp(qp), request_idr(),
set_gop(n), resize(src_w, src_h, dst_w, dst_h), flush().  The GPU side submits without flushing unless a flush() event asks
for it, so pictures stay in flight on both streams as they do in a live session; control calls land between two submits
(include/b2video.h: a call made after submit k applies from picture k+1).  Pictures enter through the host ring
(Config.entry "ring") or, as bench.py feeds them, as frames resident on the device ("resident": each distinct frame object is
uploaded once).  The oracle side restates the host rules of b2v_api.cu: the per-picture target int(kbps * 1000 / fps), the IDR
decision `want_idr or (gop > 0 and frames_since_idr >= gop)`, and a resize = a fresh encoder at the new size fed the oracle's
CSC(+scale), starting with an IDR.

Per picture, every delivered band (one band at y_start 0 in full-frame mode) must equal the oracle's: bytes, is_key, qp,
frame_id, y_start and height, and in pixelflux header mode the 10-byte header that carries them.  At the end of every segment
(the pictures between two resizes) the reconstructions must be equal and libavcodec must decode the segment's stream (every
band's stream on its own in striped mode) to that reconstruction."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Iterable, Optional

import numpy as np

import oracle
from oracle import avdec


def picture(frame):
    return ("picture", frame)


def set_bitrate(kbps):
    return ("set_bitrate", int(kbps))


def set_fps(fps):
    return ("set_fps", float(fps))


def set_qp(qp):
    return ("set_qp", int(qp))


def request_idr():
    return ("request_idr",)


def set_gop(n):
    return ("set_gop", int(n))


def resize(src_w, src_h, dst_w=0, dst_h=0):
    return ("resize", int(src_w), int(src_h), int(dst_w or src_w), int(dst_h or src_h))


def flush():
    return ("flush",)


def stream(frames, idr_at=()) -> list:
    """Pictures of `frames` in order, with flush() and request_idr() before every picture index in idr_at except 0."""
    events = []
    for i, f in enumerate(frames):
        if i in idr_at and i > 0:
            events += [flush(), request_idr()]
        events.append(picture(f))
    return events


def describe(ev) -> str:
    return ev[0] + "(" + ", ".join(str(a) for a in ev[1:]) + ")"


CBR, CQP = 0, 1                  # = selkies_b200._native.B2V_RC_CBR / B2V_RC_CQP (the oracle side needs no library)
HDR_NONE, HDR_PIXELFLUX = 0, 1   # = selkies_b200._native.B2V_HDR_NONE / B2V_HDR_PIXELFLUX


@dataclass
class Config:
    width: int
    height: int
    dst_width: int = 0
    dst_height: int = 0
    rc_mode: int = CQP
    qp: int = 28
    kbps: int = 8000
    fps: float = 60.0
    gop: int = -1
    paint: tuple = (0, 18, 1)          # (trigger pictures, paint-over QP, burst pictures); trigger 0 = off
    stripe_rows: int = 0
    slice_rows: int = 0                # 0 = the default rule (8-row slices), as in Session and RefEncoder
    idr_slice_mbs: int = 0
    header_mode: int = HDR_NONE
    flags: int = 0                     # B2V_FLAG_* bits of the GPU session
    ring_slots: int = 4
    entry: str = "ring"                # "ring" (b2v_ring_submit) or "resident" (b2v_resident_upload + b2v_submit_resident)


@dataclass
class Expected:
    index: int                         # picture index in the whole stream (= frame_id)
    is_key: bool
    qp: int
    target_bits: int
    bands: list                        # [(y_start, bytes)]: one entry at y_start 0 in full-frame mode
    rc: dict                           # oracle rate-control record after this picture (RefEncoder.rc_state)
    after: str                         # the control event just before this picture (or "start")

    @property
    def au(self) -> bytes:
        """The access unit of a full-frame picture."""
        (_, au), = self.bands
        return au


@dataclass
class Segment:
    dst: tuple                         # (dst_w, dst_h)
    first: int                         # index of its first picture
    pictures: list = field(default_factory=list)       # [Expected]


class OracleSide:
    def __init__(self, cfg: Config):
        self.cfg = cfg
        self.kbps, self.fps, self.qp, self.gop = cfg.kbps, cfg.fps, cfg.qp, cfg.gop
        self.want_idr, self.frames_since_idr, self.frame_id = True, 0, 0
        self._new_encoder(cfg.width, cfg.height, cfg.dst_width or cfg.width, cfg.dst_height or cfg.height)

    def _new_encoder(self, sw, sh, dw, dh):
        self.src, self.dst = (sw, sh), (dw, dh)
        self.enc = oracle.RefEncoder(dw, dh, self.cfg.slice_rows)
        self.enc.set_idr_slice_mbs(self.cfg.idr_slice_mbs)
        if self.cfg.stripe_rows:
            self.enc.set_stripes(self.cfg.stripe_rows)
        if self.cfg.paint[0] > 0:
            self.enc.set_paintover(*self.cfg.paint)

    def control(self, ev):
        kind = ev[0]
        if kind == "set_bitrate":
            self.kbps = ev[1]
        elif kind == "set_fps":
            self.fps = ev[1]
        elif kind == "set_qp":
            self.qp = ev[1]
        elif kind == "set_gop":
            self.gop = ev[1]
        elif kind == "request_idr":
            self.want_idr = True
        elif kind == "resize":
            self._new_encoder(*ev[1:])
            self.want_idr = True
        elif kind != "flush":          # the oracle has nothing in flight
            raise ValueError(f"unknown event {ev!r}")

    def picture(self, frame, after: str) -> Expected:
        assert frame.shape == (self.src[1], self.src[0], 4), (frame.shape, self.src)
        idr = self.want_idr or (self.gop > 0 and self.frames_since_idr >= self.gop)
        self.want_idr = False
        self.frames_since_idr = 1 if idr else self.frames_since_idr + 1
        target = int(self.kbps * 1000.0 / self.fps)
        e = self.enc
        y, uv = oracle.csc_nv12(frame, self.dst[0], self.dst[1], e.cw, e.ch)
        au = e.encode_nv12(y, uv, idr, rc_mode=self.cfg.rc_mode, qp=self.qp, target_bits=target)
        if self.cfg.stripe_rows:
            bands = [(k * self.cfg.stripe_rows * 16, au[o:o + sz]) for k, (o, sz, coded) in enumerate(e.stripe_table()) if coded]
        else:
            bands = [(0, au)]
        x = Expected(self.frame_id, idr, e.last_qp, target, bands, e.rc_state(), after)
        self.frame_id += 1
        return x


class GpuSide:
    def __init__(self, cfg: Config, device: int = 0):
        from selkies_b200.session import Session
        assert cfg.entry in ("ring", "resident"), cfg.entry
        p = cfg.paint
        self.resident = cfg.entry == "resident"
        self.uploaded = {}                 # id(frame) -> (resident index, frame); the frame is held so that its id stays unique
        self.s = Session(cfg.width, cfg.height, dst_width=cfg.dst_width, dst_height=cfg.dst_height, fps=cfg.fps, device=device,
                         rc_mode=cfg.rc_mode, bitrate_kbps=cfg.kbps, crf=cfg.qp, gop=cfg.gop, slice_rows=cfg.slice_rows,
                         idr_slice_mbs=cfg.idr_slice_mbs, stripe_rows=cfg.stripe_rows, header_mode=cfg.header_mode,
                         paintover_trigger_frames=p[0], paintover_crf=p[1], paintover_burst_frames=p[2], ring_slots=cfg.ring_slots,
                         flags=cfg.flags)

    def control(self, ev):
        kind, s = ev[0], self.s
        if kind == "set_bitrate":
            s.set_bitrate_kbps(ev[1])
        elif kind == "set_fps":
            s.set_framerate(ev[1])
        elif kind == "set_qp":
            s.set_qp(ev[1])
        elif kind == "set_gop":
            s.set_gop(ev[1])
        elif kind == "request_idr":
            s.request_idr()
        elif kind == "flush":
            s.flush()
        elif kind == "resize":
            s.set_resolution(*ev[1:])
            self.uploaded.clear()          # the library frees its resident frames on a resize

    def picture(self, frame):
        if not self.resident:
            self.s.submit(frame)           # no flush: the picture stays in flight
            return
        if id(frame) not in self.uploaded:
            k = len(self.uploaded)
            self.s.resident_upload(k, frame)
            self.uploaded[id(frame)] = (k, frame)
        self.s.submit_resident(self.uploaded[id(frame)][0])


def _first_diff(a: bytes, b: bytes) -> int:
    n = min(len(a), len(b))
    return next((k for k in range(n) if a[k] != b[k]), n)


def _where(x: Expected) -> str:
    return f"picture {x.index} (after {x.after})"


def _band_height(cfg: Config, h: int, y0: int) -> int:
    return min(h, y0 + cfg.stripe_rows * 16) - y0 if cfg.stripe_rows else h


def _check_segment(cfg: Config, seg: Segment, got: list, grec, rrec, decode: bool):
    w, h = seg.dst
    if cfg.stripe_rows:
        per = {}
        for g in got:
            per.setdefault(g.frame_id, []).append(g)
        assert set(per) <= {x.index for x in seg.pictures}, f"bands delivered for pictures outside the segment: {sorted(per)}"
    else:
        assert len(got) == len(seg.pictures), f"segment at picture {seg.first}: {len(got)} access units for {len(seg.pictures)} pictures"
        per = {x.index: [g] for x, g in zip(seg.pictures, got)}
    for x in seg.pictures:
        gs = per.get(x.index, [])
        where = _where(x)
        assert len(gs) == len(x.bands), f"{where}: {len(gs)} bands delivered, oracle codes {len(x.bands)} (y_start {[y for y, _ in x.bands]})"
        for g, (y0, ref) in zip(gs, x.bands):
            bh = _band_height(cfg, h, y0)
            assert g.frame_id == x.index, f"{where}: frame_id {g.frame_id}"
            assert g.is_key == x.is_key, f"{where}: is_key gpu {g.is_key} oracle {x.is_key}"
            assert g.qp == x.qp, f"{where}: qp gpu {g.qp} oracle {x.qp}"
            assert g.y_start == y0, f"{where}: band y_start gpu {g.y_start} oracle {y0}"
            assert g.height == bh, f"{where}, band y_start {y0}: height gpu {g.height}, expected {bh}"
            data = g.data
            if cfg.header_mode == HDR_PIXELFLUX:
                # 04 | is_key | frame_id u16be | y_start u16be | width u16be | band height u16be
                hdr = bytes([4, x.is_key]) + b"".join(v.to_bytes(2, "big") for v in (x.index & 0xFFFF, y0, w, bh))
                assert data[:10] == hdr, f"{where}, band y_start {y0}: header {data[:10].hex()}, expected {hdr.hex()}"
                data = data[10:]
            if data != ref:
                raise AssertionError(f"{where}, band y_start {y0}: AU differs at byte {_first_diff(data, ref)} "
                                     f"(gpu {len(data)} B, oracle {len(ref)} B, qp {g.qp})")
    first = seg.pictures[0]
    assert first.is_key, f"segment at picture {seg.first} does not start with an IDR"
    for _, au in first.bands:
        assert au[:5] == b"\x00\x00\x00\x01\x67", f"segment at picture {seg.first}: first access unit carries no SPS"
    assert np.array_equal(grec[0], rrec[0]) and np.array_equal(grec[1], rrec[1]), f"segment at picture {seg.first}: reconstruction differs"
    if not decode:
        return
    bands = sorted({y0 for x in seg.pictures for y0, _ in x.bands})
    for y0 in bands:
        y1 = y0 + _band_height(cfg, h, y0)
        aus = [au for x in seg.pictures for yb, au in x.bands if yb == y0]
        dec = avdec.decode_stream(aus, quiet=True)
        assert len(dec) == len(aus), f"segment at picture {seg.first}, band {y0}: {len(dec)} pictures decoded of {len(aus)}"
        Y, U, V = dec[-1]
        assert Y.shape == (y1 - y0, w), f"segment at picture {seg.first}: decoded size {Y.shape[::-1]}, expected {(w, y1 - y0)}"
        assert np.array_equal(Y, grec[0][y0:y1, :w]), f"segment at picture {seg.first}, band {y0}: decoded luma != reconstruction"
        assert np.array_equal(U, grec[1][y0 // 2:y1 // 2, 0:w:2]) and np.array_equal(V, grec[1][y0 // 2:y1 // 2, 1:w:2]), \
            f"segment at picture {seg.first}, band {y0}: decoded chroma != reconstruction"


def run(cfg: Config, events: Iterable, *, gpu: bool = True, decode: bool = True, device: int = 0) -> list:
    """Apply `events` to the oracle and (gpu=True) to a GPU session; compare as described above.  Returns the segments, each with
    the oracle's Expected record of every picture (bytes, qp, rate-control state), for assertions of the caller."""
    o = OracleSide(cfg)
    g: Optional[GpuSide] = GpuSide(cfg, device) if gpu else None
    segs = [Segment(o.dst, 0)]
    after = "start"

    def close_segment():
        seg = segs[-1]
        if g is None or not seg.pictures:
            return
        grec = g.s.recon()                 # waits for the segment's last picture
        _check_segment(cfg, seg, g.s.take_frames(), grec, o.enc.recon(), decode)

    try:
        for ev in events:
            if ev[0] == "picture":
                x = o.picture(ev[1], after)
                segs[-1].pictures.append(x)
                if g is not None:
                    g.picture(ev[1])
                continue
            if ev[0] == "resize":
                close_segment()
            o.control(ev)
            if g is not None:
                g.control(ev)
            after = f"{describe(ev)} before picture {o.frame_id}"
            if ev[0] == "resize":
                segs.append(Segment(o.dst, o.frame_id))
        close_segment()
    finally:
        if g is not None:
            g.s.close()
    return [s for s in segs if s.pictures]


def pictures(segs) -> list:
    """Every picture's Expected record, in stream order."""
    return [x for s in segs for x in s.pictures]
