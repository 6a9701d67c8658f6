"""GPU parity: the fused CSC(+scale) kernel vs oracle/csc_ref.c, bit-exact, through the C-ABI."""
import numpy as np
import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import synth

pytestmark = pytest.mark.gpu

SIZES = [(16, 16), (64, 48), (128, 2), (130, 34), (1920, 1080), (3840, 2160), (258, 66)]


@pytest.mark.parametrize("w,h", [s for s in SIZES if s[1] >= 16])
def test_csc_bit_exact(w, h):
    frames = [synth.noise(w, h, 11), synth.bars(w, h, 3), synth.gradient(w, h, 5)]
    with Session(w, h, flags=N.B2V_FLAG_NO_ENCODE) as s:
        for f in frames:
            y, uv = s.csc_nv12(f)
            oy, ouv = oracle.csc_nv12(f)
            assert np.array_equal(y, oy)
            assert np.array_equal(uv, ouv)


@pytest.mark.parametrize("sw,sh,dw,dh", [(320, 180, 192, 108), (640, 360, 1280, 720), (1920, 1080, 1280, 720), (100, 60, 64, 48)])
def test_csc_scaled_bit_exact(sw, sh, dw, dh):
    f = synth.noise(sw, sh, 21)
    with Session(sw, sh, dst_width=dw, dst_height=dh, flags=N.B2V_FLAG_NO_ENCODE) as s:
        y, uv = s.csc_nv12(f)
    oy, ouv = oracle.csc_nv12(f, dst_w=dw, dst_h=dh)
    assert np.array_equal(y, oy)
    assert np.array_equal(uv, ouv)


def test_csc_extremes():
    w, h = 64, 32
    for v in (0, 255):
        f = np.full((h, w, 4), v, np.uint8)
        with Session(w, h, flags=N.B2V_FLAG_NO_ENCODE) as s:
            y, uv = s.csc_nv12(f)
        oy, ouv = oracle.csc_nv12(f)
        assert np.array_equal(y, oy) and np.array_equal(uv, ouv)


def test_csc_8k_property():
    """BASELINE config 4 size: checksum-of-tiles property instead of a full oracle run."""
    w, h = 7680, 4320
    tile = synth.noise(256, 144, 31)
    f = np.tile(tile, (h // 144, w // 256, 1))
    with Session(w, h, flags=N.B2V_FLAG_NO_ENCODE) as s:
        y, uv = s.csc_nv12(f)
    oy, ouv = oracle.csc_nv12(tile)
    assert np.array_equal(y, np.tile(oy, (h // 144, w // 256)))
    assert np.array_equal(uv, np.tile(ouv, (h // 144, w // 256)))


@pytest.mark.parametrize("sw,sh,dw,dh", [(3840, 2160, 1920, 1080), (1920, 1080, 3840, 2160), (1922, 1082, 1280, 720), (640, 360, 2560, 1440), (1280, 720, 1276, 716)])
def test_csc_scaled_tiled_bit_exact_large(sw, sh, dw, dh):
    """The shared-memory-tiled scale+CSC kernel at the sizes bench.py times (4K <-> 1080p), a source width that is not a
    multiple of 4, a 4x upscale and a near-1:1 ratio."""
    f = synth.noise(sw, sh, 5)
    with Session(sw, sh, dst_width=dw, dst_height=dh, flags=N.B2V_FLAG_NO_ENCODE) as s:
        y, uv = s.csc_nv12(f)
    oy, ouv = oracle.csc_nv12(f, dst_w=dw, dst_h=dh)
    assert np.array_equal(y, oy)
    assert np.array_equal(uv, ouv)


@pytest.mark.parametrize("sw,sh,dw,dh", [(1920, 1080, 320, 180), (7680, 4320, 1280, 720)])
def test_csc_scaled_tiled_opt_in_shared_memory_tier(sw, sh, dw, dh):
    """Downscales by 6: the tiled kernel's source footprint is 392 x 51 pixels (80 KB), above the 48 KB a launch gets without
    the opt-in attribute."""
    f = synth.noise(sw, sh, 9)
    with Session(sw, sh, dst_width=dw, dst_height=dh, flags=N.B2V_FLAG_NO_ENCODE) as s:
        y, uv = s.csc_nv12(f)
    oy, ouv = oracle.csc_nv12(f, dst_w=dw, dst_h=dh)
    assert np.array_equal(y, oy)
    assert np.array_equal(uv, ouv)


def test_csc_scaled_close_to_cv2_resize():
    """SURVEY §8c.3: the fused bilinear scale stays within rounding distance of cv2.resize(INTER_LINEAR) followed by the 1:1
    conversion (cv2 blends with 11-bit weights, this spec with 8-bit ones: +-1 per channel before the matrix)."""
    cv2 = pytest.importorskip("cv2")
    sw, sh, dw, dh = 1920, 1080, 1280, 720
    f = synth.gradient(sw, sh, 3)
    f[200:400, 300:900] = synth.noise(600, 200, 4)
    with Session(sw, sh, dst_width=dw, dst_height=dh, flags=N.B2V_FLAG_NO_ENCODE) as s:
        y, uv = s.csc_nv12(f)
    ref = np.ascontiguousarray(cv2.resize(f, (dw, dh), interpolation=cv2.INTER_LINEAR))
    ry, ruv = oracle.csc_nv12(ref)
    dy = np.abs(y.astype(int) - ry.astype(int))
    assert dy.max() <= 1
    assert np.abs(uv.astype(int) - ruv.astype(int)).max() <= 1
