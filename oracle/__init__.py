"""CPU oracle for the video hot path — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this package.  Nothing under selkies_b200/ does (tests/test_boundary.py enforces it).

PARITY UNPINNED: see the headers of csc_ref.c and h264_ref.c — the reference tree holds neither an
implementation nor golden vectors for this path.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "_build", "liboracle.so")
_lib = None


def build(force: bool = False) -> str:
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".c", ".h"))]
    stale = (not os.path.exists(_LIB)) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in srcs)
    if force or stale:
        subprocess.check_call(["make", "-s", "-C", _HERE])
    return _LIB


def lib():
    global _lib
    if _lib is None:
        try:
            build()
        except Exception:
            if not os.path.exists(_LIB):
                raise
        _lib = C.CDLL(_LIB)
    return _lib


def set_threads(n: int = 0) -> int:
    """Host threads for the oracle's OpenMP loops (0 = all cores); returns the count in effect."""
    L = lib()
    L.b2v_ref_set_threads(int(n))
    return int(L.b2v_ref_max_threads())


def _u8p(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint8))


def csc_nv12(bgra: np.ndarray, dst_w: int = 0, dst_h: int = 0, coded_w: int = 0, coded_h: int = 0, matrix: int = 0):
    """BGRA (H,W,4) uint8 -> (Y (coded_h,coded_w), UV (coded_h/2,coded_w)) per oracle/csc_ref.c.
    matrix 0 = BT.709 limited range (H.264 path), 1 = JFIF full-range BT.601 (JPEG stripe path)."""
    assert bgra.dtype == np.uint8 and bgra.ndim == 3 and bgra.shape[2] == 4
    bgra = np.ascontiguousarray(bgra)
    sh, sw = bgra.shape[:2]
    dst_w = dst_w or sw
    dst_h = dst_h or sh
    coded_w = coded_w or dst_w
    coded_h = coded_h or dst_h
    y = np.empty((coded_h, coded_w), np.uint8)
    uv = np.empty((coded_h // 2, coded_w), np.uint8)
    rc = lib().b2v_ref_csc_nv12_m(_u8p(bgra), sw, sh, sw * 4, dst_w, dst_h, coded_w, coded_h, _u8p(y), _u8p(uv), matrix)
    if rc != 0:
        raise ValueError(f"b2v_ref_csc_nv12 rc={rc}")
    return y, uv


def jpeg_encode(y: np.ndarray, uv, width: int, height: int, quality: int) -> bytes:
    """One baseline JFIF file per oracle/jpeg_ref.c.  y: (H',W') luma rows, uv: (H'/2, W') interleaved Cb,Cr rows or None (grey);
    H', W' >= the next multiple of 16 (8 when grey) of height, width (padded by replication by the caller)."""
    L = lib()
    L.b2v_ref_jpeg_encode.restype = C.c_int64
    L.b2v_ref_jpeg_encode.argtypes = [C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint8)]
    y = np.ascontiguousarray(y)
    pitch = y.shape[1]
    out = np.empty(y.size * 3 + 4096, np.uint8)
    if uv is not None:
        uv = np.ascontiguousarray(uv)
        assert uv.shape[1] == pitch
    n = L.b2v_ref_jpeg_encode(_u8p(y), _u8p(uv) if uv is not None else None, pitch, width, height, quality, _u8p(out))
    return out[:n].tobytes()


def jpeg_encode_bgra(bgra: np.ndarray, quality: int) -> bytes:
    """oracle CSC (JFIF matrix, padded to a multiple of 16) + oracle JPEG: what one stripe of the JPEG mode must equal."""
    h, w = bgra.shape[:2]
    cw, ch = (w + 15) & ~15, (h + 15) & ~15
    y, uv = csc_nv12(bgra, coded_w=cw, coded_h=ch, matrix=1)
    return jpeg_encode(y, uv, w, h, quality)


class RefEncoder:
    """ctypes wrapper of oracle/h264_ref.c (one encoder instance)."""

    def __init__(self, width: int, height: int, slice_rows: int = 0):
        L = lib()
        L.b2v_ref_enc_create.restype = C.c_void_p
        L.b2v_ref_enc_create.argtypes = [C.c_int, C.c_int, C.c_int]
        L.b2v_ref_enc_destroy.argtypes = [C.c_void_p]
        L.b2v_ref_enc_coded_w.argtypes = [C.c_void_p]
        L.b2v_ref_enc_coded_h.argtypes = [C.c_void_p]
        L.b2v_ref_enc_recon.restype = C.POINTER(C.c_uint8)
        L.b2v_ref_enc_recon.argtypes = [C.c_void_p]
        L.b2v_ref_enc_last_qp.argtypes = [C.c_void_p]
        L.b2v_ref_enc_max_au.restype = C.c_size_t
        L.b2v_ref_enc_max_au.argtypes = [C.c_void_p]
        L.b2v_ref_enc_encode.restype = C.c_int64
        L.b2v_ref_enc_encode.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, C.c_int64, C.POINTER(C.c_uint8)]
        self.L = L
        self.width, self.height = width, height
        self.h = C.c_void_p(L.b2v_ref_enc_create(width, height, slice_rows))
        self.cw, self.ch = L.b2v_ref_enc_coded_w(self.h), L.b2v_ref_enc_coded_h(self.h)
        self._out = np.empty(L.b2v_ref_enc_max_au(self.h), np.uint8)
        L.b2v_ref_enc_set_paintover.argtypes = [C.c_void_p, C.c_int, C.c_int]

    def set_stripes(self, stripe_rows: int) -> int:
        """Striped mode: bands of `stripe_rows` macroblock rows, each an independent stream.  Returns the band count."""
        self.L.b2v_ref_enc_set_stripes.argtypes = [C.c_void_p, C.c_int]
        n = self.L.b2v_ref_enc_set_stripes(self.h, stripe_rows)
        if n < 0:
            raise ValueError("stripe_rows must be a multiple of slice_rows")
        self.stripe_rows = stripe_rows if n > 1 else 0
        return n

    def stripe_table(self):
        """[(offset, size, coded)] per band for the last picture (empty when striping is off)."""
        t = np.zeros(512 * 3, np.int32)
        self.L.b2v_ref_enc_stripe_table.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
        n = self.L.b2v_ref_enc_stripe_table(self.h, t.ctypes.data_as(C.POINTER(C.c_int32)))
        return [tuple(int(v) for v in t[3 * i: 3 * i + 3]) for i in range(n)]

    def set_idr_slice_mbs(self, n: int) -> None:
        """Slices of IDR pictures: n > 0 macroblocks per slice inside a row, n < 0 whole rows, 0 = the default rule."""
        self.L.b2v_ref_enc_set_idr_slice_mbs.argtypes = [C.c_void_p, C.c_int]
        self.L.b2v_ref_enc_set_idr_slice_mbs(self.h, n)

    def set_paintover(self, trigger_frames: int, qp: int, burst_frames: int = 1) -> None:
        self.L.b2v_ref_enc_set_paintover(self.h, trigger_frames, qp)
        self.L.b2v_ref_enc_set_paintover_burst.argtypes = [C.c_void_p, C.c_int]
        self.L.b2v_ref_enc_set_paintover_burst(self.h, burst_frames)

    def encode_nv12(self, y: np.ndarray, uv: np.ndarray, idr: bool, rc_mode: int = 1, qp: int = 26, target_bits: int = 0) -> bytes:
        assert y.shape == (self.ch, self.cw) and uv.shape == (self.ch // 2, self.cw)
        cur = np.concatenate([y.reshape(-1), uv.reshape(-1)])
        n = self.L.b2v_ref_enc_encode(self.h, _u8p(cur), int(idr), rc_mode, qp, target_bits, _u8p(self._out))
        return self._out[:n].tobytes()

    def encode_bgra(self, bgra: np.ndarray, idr: bool, **kw) -> bytes:
        """oracle CSC (with padding to the coded size) + oracle encode."""
        y, uv = csc_nv12(bgra, dst_w=self.width, dst_h=self.height, coded_w=self.cw, coded_h=self.ch)
        return self.encode_nv12(y, uv, idr, **kw)

    def recon(self):
        p = self.L.b2v_ref_enc_recon(self.h)
        a = np.ctypeslib.as_array(p, shape=(self.cw * self.ch * 3 // 2,)).copy()
        return a[: self.cw * self.ch].reshape(self.ch, self.cw), a[self.cw * self.ch:].reshape(self.ch // 2, self.cw)

    @property
    def last_qp(self):
        return self.L.b2v_ref_enc_last_qp(self.h)

    def rc_state(self) -> dict:
        """The rate-control / paint-over record written after the last picture: fullness (bits), qp (decided for a later
        picture), static_run, remaining (paint-over pictures still to schedule), paint, debt (the debt rule raised the QP)."""
        v = np.zeros(6, np.int64)
        self.L.b2v_ref_enc_rc_state.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        if self.L.b2v_ref_enc_rc_state(self.h, v.ctypes.data_as(C.POINTER(C.c_int64))) != 0:
            raise ValueError("no picture encoded yet")
        return dict(zip(("fullness", "qp", "static_run", "remaining", "paint", "debt"), (int(x) for x in v)))

    def close(self):
        if self.h:
            self.L.b2v_ref_enc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
