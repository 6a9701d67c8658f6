"""Wide-range motion (B2V_FLAG_WIDE_MOTION) in the CPU oracle — TEST INFRASTRUCTURE ONLY: oracle/h264_wide_ref.c around the
single-layer encoder of oracle/h264_ref.c, droppable through the layers of oracle/h264_layers_ref.c."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _u8p
from .layers import LayeredRefEncoder

COARSE_NONE = 0x7fffffff         # h264_wide_ref.c: an anchor group without a coarse vector, and every other macroblock


class WideRefEncoder(LayeredRefEncoder):
    """LayeredRefEncoder with wide-range motion once set_wide_motion(True) is called (before the first picture; droppable pictures
    and stripes are set before it too); without it, exactly LayeredRefEncoder."""

    def __init__(self, width: int, height: int, slice_rows: int = 0):
        super().__init__(width, height, slice_rows)
        self.wide_motion = False
        self._wide = None

    def set_wide_motion(self, on: bool) -> None:
        if not on:
            if self.wide_motion:
                raise ValueError("wide motion cannot be turned off")
            return
        if self._wide is None:
            L = self.L
            L.b2v_ref_wide_create.restype = C.c_void_p
            L.b2v_ref_wide_create.argtypes = [C.c_void_p, C.c_int]
            L.b2v_ref_wide_destroy.argtypes = [C.c_void_p]
            L.b2v_ref_wide_encode.restype = C.c_int64
            L.b2v_ref_wide_encode.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, C.c_int64,
                                              C.POINTER(C.c_uint8)]
            self._wide = C.c_void_p(L.b2v_ref_wide_create(self.h, int(self.droppable)))
        self.wide_motion = True

    def set_droppable(self, on: bool) -> None:
        if self.wide_motion and on != self.droppable:
            raise ValueError("set droppable pictures before wide motion")
        super().set_droppable(on)

    def set_stripes(self, stripe_rows: int) -> int:
        if self.wide_motion:
            raise ValueError("set stripes before wide motion")
        return super().set_stripes(stripe_rows)

    def encode_nv12(self, y: np.ndarray, uv: np.ndarray, idr: bool, rc_mode: int = 1, qp: int = 26, target_bits: int = 0) -> bytes:
        if not self.wide_motion:
            return super().encode_nv12(y, uv, idr, rc_mode, qp, target_bits)
        assert y.shape == (self.ch, self.cw) and uv.shape == (self.ch // 2, self.cw)
        cur = np.concatenate([y.reshape(-1), uv.reshape(-1)])
        n = self.L.b2v_ref_wide_encode(self._wide, _u8p(cur), int(idr), rc_mode, qp, target_bits, _u8p(self._out))
        return self._out[:n].tobytes()

    def coarse(self) -> list:
        """The last picture's coarse vectors: coarse()[mby][mbx] is (dx, dy) in decimated samples at an anchor whose group has one,
        None elsewhere (every macroblock of an IDR picture)."""
        assert self.wide_motion
        mbw, mbh = self.cw // 16, self.ch // 16
        t = np.empty(mbw * mbh, np.int32)
        self.L.b2v_ref_wide_coarse.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
        self.L.b2v_ref_wide_coarse(self._wide, t.ctypes.data_as(C.POINTER(C.c_int32)))
        return [[None if v == COARSE_NONE else (int(np.int16(v & 0xffff)), int(v >> 16)) for v in row] for row in t.reshape(mbh, mbw)]

    def decimated(self) -> np.ndarray:
        """The last picture's decimated luma plane, (ch / 4) x (cw / 4)."""
        assert self.wide_motion
        d = np.empty((self.ch // 4, self.cw // 4), np.uint8)
        self.L.b2v_ref_wide_decimated.argtypes = [C.c_void_p, C.POINTER(C.c_uint8)]
        self.L.b2v_ref_wide_decimated(self._wide, _u8p(d))
        return d

    def close(self):
        if getattr(self, "_wide", None):
            self.L.b2v_ref_wide_destroy(self._wide)
            self._wide = None
        super().close()
