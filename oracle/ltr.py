"""The long-term reference picture (B2V_FLAG_LONG_TERM_REF) in the CPU oracle — TEST INFRASTRUCTURE ONLY: oracle/h264_ltr_ref.c around
the single-layer encoder of oracle/h264_ref.c, with or without the wide-range motion of oracle/h264_wide_ref.c."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _u8p
from .wide import WideRefEncoder


class LongTermRefEncoder(WideRefEncoder):
    """WideRefEncoder with a long-term reference picture once set_long_term_ref(True) is called (before the first picture, after
    set_wide_motion; full frame only, no droppable pictures); without it, exactly WideRefEncoder."""

    def __init__(self, width: int, height: int, slice_rows: int = 0):
        super().__init__(width, height, slice_rows)
        self.long_term_ref = False
        self._ltr = None

    def set_long_term_ref(self, on: bool) -> None:
        if not on:
            if self.long_term_ref:
                raise ValueError("the long-term reference cannot be turned off")
            return
        if self.droppable or getattr(self, "stripe_rows", 0):
            raise ValueError("the long-term reference is full-frame only, without droppable pictures")
        L = self.L
        L.b2v_ref_ltr_create.restype = C.c_void_p
        L.b2v_ref_ltr_create.argtypes = [C.c_void_p, C.c_int]
        L.b2v_ref_ltr_destroy.argtypes = [C.c_void_p]
        L.b2v_ref_ltr_encode.restype = C.c_int64
        L.b2v_ref_ltr_encode.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, C.c_int64, C.POINTER(C.c_uint8)]
        L.b2v_ref_ltr_state.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
        L.b2v_ref_ltr_picture.restype = C.POINTER(C.c_uint8)
        L.b2v_ref_ltr_picture.argtypes = [C.c_void_p]
        self._ltr = C.c_void_p(L.b2v_ref_ltr_create(self.h, int(self.wide_motion)))
        self.long_term_ref = True

    def set_wide_motion(self, on: bool) -> None:
        if self.long_term_ref:
            raise ValueError("set wide motion before the long-term reference")
        super().set_wide_motion(on)

    def set_droppable(self, on: bool) -> None:
        if self.long_term_ref and on:
            raise ValueError("droppable pictures cannot mark a long-term picture")
        super().set_droppable(on)

    def encode_nv12(self, y: np.ndarray, uv: np.ndarray, idr: bool, rc_mode: int = 1, qp: int = 26, target_bits: int = 0) -> bytes:
        if not self.long_term_ref:
            return super().encode_nv12(y, uv, idr, rc_mode, qp, target_bits)
        assert y.shape == (self.ch, self.cw) and uv.shape == (self.ch // 2, self.cw)
        cur = np.concatenate([y.reshape(-1), uv.reshape(-1)])
        n = self.L.b2v_ref_ltr_encode(self._ltr, _u8p(cur), int(idr), rc_mode, qp, target_bits, _u8p(self._out))
        return self._out[:n].tobytes()

    def ltr_state(self) -> dict:
        """The last picture: two active references, marks the previous picture long-term, MMCO 1 first, changed(k)."""
        v = np.zeros(4, np.int32)
        self.L.b2v_ref_ltr_state(self._ltr, v.ctypes.data_as(C.POINTER(C.c_int32)))
        return dict(zip(("active", "mark", "drop_st", "changed"), (int(x) for x in v)))

    def long_term_picture(self):
        """(Y, UV) of the long-term reference picture as the next picture sees it, or None while there is none."""
        p = self.L.b2v_ref_ltr_picture(self._ltr)
        if not p:
            return None
        a = np.ctypeslib.as_array(p, shape=(self.cw * self.ch * 3 // 2,)).copy()
        return a[: self.cw * self.ch].reshape(self.ch, self.cw), a[self.cw * self.ch:].reshape(self.ch // 2, self.cw)

    def close(self):
        if getattr(self, "_ltr", None):
            self.L.b2v_ref_ltr_destroy(self._ltr)
            self._ltr = None
        super().close()
