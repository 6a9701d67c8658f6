"""Droppable pictures (B2V_FLAG_DROPPABLE) in the CPU oracle — TEST INFRASTRUCTURE ONLY: oracle/h264_layers_ref.c around the
single-layer encoder of oracle/h264_ref.c."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import RefEncoder, _u8p


class LayeredRefEncoder(RefEncoder):
    """RefEncoder with two temporal layers once set_droppable(True) is called (before the first picture); without it, exactly
    RefEncoder.  Full frame only: the combination with stripes is refused either way round."""

    def __init__(self, width: int, height: int, slice_rows: int = 0):
        super().__init__(width, height, slice_rows)
        self.droppable = False
        self._layers = None

    def set_droppable(self, on: bool) -> None:
        L = self.L
        if not on:
            self.droppable = False
            return
        if getattr(self, "stripe_rows", 0):
            raise ValueError("droppable pictures are full-frame only: striped mode is on")
        if self._layers is None:
            L.b2v_ref_layers_create.restype = C.c_void_p
            L.b2v_ref_layers_create.argtypes = [C.c_void_p]
            L.b2v_ref_layers_destroy.argtypes = [C.c_void_p]
            L.b2v_ref_layers_encode.restype = C.c_int64
            L.b2v_ref_layers_encode.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, C.c_int64,
                                                C.POINTER(C.c_uint8)]
            self._layers = C.c_void_p(L.b2v_ref_layers_create(self.h))
        self.droppable = True

    def set_stripes(self, stripe_rows: int) -> int:
        if self.droppable and 0 < stripe_rows < self.ch // 16:
            raise ValueError("droppable pictures are full-frame only")
        return super().set_stripes(stripe_rows)

    def encode_nv12(self, y: np.ndarray, uv: np.ndarray, idr: bool, rc_mode: int = 1, qp: int = 26, target_bits: int = 0) -> bytes:
        if not self.droppable:
            return super().encode_nv12(y, uv, idr, rc_mode, qp, target_bits)
        assert y.shape == (self.ch, self.cw) and uv.shape == (self.ch // 2, self.cw)
        cur = np.concatenate([y.reshape(-1), uv.reshape(-1)])
        n = self.L.b2v_ref_layers_encode(self._layers, _u8p(cur), int(idr), rc_mode, qp, target_bits, _u8p(self._out))
        return self._out[:n].tobytes()

    def close(self):
        if getattr(self, "_layers", None):
            self.L.b2v_ref_layers_destroy(self._layers)
            self._layers = None
        super().close()
