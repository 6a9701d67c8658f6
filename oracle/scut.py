"""Scene cuts (B2V_FLAG_SCENE_CUT) in the CPU oracle — TEST INFRASTRUCTURE ONLY: oracle/h264_scut_ref.c around the single-layer encoder
of oracle/h264_ref.c, with any permitted combination of droppable pictures, wide-range motion and the long-term reference."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _u8p
from .ltr import LongTermRefEncoder


class SceneCutEncoder(LongTermRefEncoder):
    """LongTermRefEncoder with scene cuts once set_scene_cut(True) is called (before the first picture, after every other setting;
    full frame only); without it, exactly LongTermRefEncoder."""

    def __init__(self, width: int, height: int, slice_rows: int = 0):
        super().__init__(width, height, slice_rows)
        self.scene_cut = False
        self._scut = None

    def set_scene_cut(self, on: bool) -> None:
        if not on:
            if self.scene_cut:
                raise ValueError("scene cuts cannot be turned off")
            return
        if getattr(self, "stripe_rows", 0):
            raise ValueError("scene cuts are full-frame only")
        L = self.L
        L.b2v_ref_scut_create.restype = C.c_void_p
        L.b2v_ref_scut_create.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.b2v_ref_scut_destroy.argtypes = [C.c_void_p]
        L.b2v_ref_scut_encode.restype = C.c_int64
        L.b2v_ref_scut_encode.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, C.c_int64, C.POINTER(C.c_uint8)]
        L.b2v_ref_scut_state.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        h = L.b2v_ref_scut_create(self.h, self._ltr if self.long_term_ref else None, int(self.wide_motion), int(self.droppable))
        if not h:
            raise ValueError("scene cuts are full-frame only")
        self._scut = C.c_void_p(h)
        self.scene_cut = True

    def set_long_term_ref(self, on: bool) -> None:
        if self.scene_cut:
            raise ValueError("set the long-term reference before scene cuts")
        super().set_long_term_ref(on)

    def set_wide_motion(self, on: bool) -> None:
        if self.scene_cut:
            raise ValueError("set wide motion before scene cuts")
        super().set_wide_motion(on)

    def set_droppable(self, on: bool) -> None:
        if self.scene_cut and on != self.droppable:
            raise ValueError("set droppable pictures before scene cuts")
        super().set_droppable(on)

    def encode_nv12(self, y: np.ndarray, uv: np.ndarray, idr: bool, rc_mode: int = 1, qp: int = 26, target_bits: int = 0) -> bytes:
        if not self.scene_cut:
            return super().encode_nv12(y, uv, idr, rc_mode, qp, target_bits)
        assert y.shape == (self.ch, self.cw) and uv.shape == (self.ch // 2, self.cw)
        cur = np.concatenate([y.reshape(-1), uv.reshape(-1)])
        n = self.L.b2v_ref_scut_encode(self._scut, _u8p(cur), int(idr), rc_mode, qp, target_bits, _u8p(self._out))
        return self._out[:n].tobytes()

    def scut_state(self) -> dict:
        """The last picture: cut, its two costs (0 for an IDR picture) and the lambda of its QP."""
        v = np.zeros(4, np.int64)
        self.L.b2v_ref_scut_state(self._scut, v.ctypes.data_as(C.POINTER(C.c_int64)))
        return dict(zip(("cut", "cost_intra", "cost_inter", "lambda"), (int(x) for x in v)))

    def close(self):
        if getattr(self, "_scut", None):
            self.L.b2v_ref_scut_destroy(self._scut)
            self._scut = None
        super().close()
