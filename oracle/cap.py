"""The picture size cap (B2V_FLAG_SIZE_CAP) in the CPU oracle — TEST INFRASTRUCTURE ONLY: oracle/h264_cap_ref.c around the single-layer
encoder of oracle/h264_ref.c, with any permitted combination of droppable pictures, wide-range motion, the long-term reference and
scene cuts."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _u8p
from .scut import SceneCutEncoder


class SizeCapEncoder(SceneCutEncoder):
    """SceneCutEncoder with the size cap once set_size_cap(True) is called (before the first picture, after every other setting,
    instead of set_scene_cut(True): scene cuts are then an argument; full frame only); without it, exactly SceneCutEncoder."""

    def __init__(self, width: int, height: int, slice_rows: int = 0):
        super().__init__(width, height, slice_rows)
        self.size_cap = False
        self.max_picture_bytes = 0
        self._cap = None

    def set_size_cap(self, on: bool, scene_cut: bool = False) -> None:
        if not on:
            return
        if self.scene_cut or getattr(self, "stripe_rows", 0):
            raise ValueError("the size cap is full-frame only, and takes scene cuts as an argument")
        L = self.L
        L.b2v_ref_cap_create.restype = C.c_void_p
        L.b2v_ref_cap_create.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.b2v_ref_cap_destroy.argtypes = [C.c_void_p]
        L.b2v_ref_cap_encode.restype = C.c_int64
        L.b2v_ref_cap_encode.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int,
                                         C.POINTER(C.c_uint8)]
        L.b2v_ref_cap_state.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        h = L.b2v_ref_cap_create(self.h, self._ltr if self.long_term_ref else None, int(self.wide_motion), int(self.droppable),
                                 int(scene_cut))
        if not h:
            raise ValueError("the size cap is full-frame only")
        self._cap = C.c_void_p(h)
        self.size_cap = True

    def encode_nv12(self, y: np.ndarray, uv: np.ndarray, idr: bool, rc_mode: int = 1, qp: int = 26, target_bits: int = 0) -> bytes:
        if not self.size_cap:
            return super().encode_nv12(y, uv, idr, rc_mode, qp, target_bits)
        assert y.shape == (self.ch, self.cw) and uv.shape == (self.ch // 2, self.cw)
        cur = np.concatenate([y.reshape(-1), uv.reshape(-1)])
        n = self.L.b2v_ref_cap_encode(self._cap, _u8p(cur), int(idr), rc_mode, qp, target_bits, int(self.max_picture_bytes),
                                      _u8p(self._out))
        return self._out[:n].tobytes()

    def cap_state(self) -> dict:
        """The last picture: recoded, the analysis's QP, the QP it was coded at, and the count in bits (0 for IDR and cut pictures)."""
        v = np.zeros(4, np.int64)
        self.L.b2v_ref_cap_state(self._cap, v.ctypes.data_as(C.POINTER(C.c_int64)))
        return dict(zip(("recoded", "qp", "qp_final", "bits"), (int(x) for x in v)))

    def close(self):
        if getattr(self, "_cap", None):
            self.L.b2v_ref_cap_destroy(self._cap)
            self._cap = None
        super().close()
