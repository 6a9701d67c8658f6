"""CPU: damage rectangles (B2V_FLAG_DAMAGE) where no GPU is needed.  b2v_damage_tiles, the map every damage submit converts by,
against the oracle's colour conversion: sound (every output sample that changes lies in a dirty tile), exact at 1:1, tight when
scaling.  The argument errors of the damage submits that return before any CUDA call, the Python rectangle normalisation, and
how ScreenCapture drives a DamageFrameSource."""
import numpy as np
import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.pixelflux_compat import DamageFrameSource, ScreenCapture
from selkies_b200.session import normalize_rects


def r16(v):
    return (v + 15) & ~15


def tiles(sw, sh, dw, dh, rects):
    tw, th = (dw + 15) // 16, (dh + 15) // 16
    m = np.full(tw * th, 7, np.uint8)
    arr, n = N.rect_array(rects)
    rc = N.lib().b2v_damage_tiles(sw, sh, dw, dh, arr, n, m.ctypes.data)
    assert rc >= 0, N.lib().b2v_last_error()
    m = m.reshape(th, tw)
    assert set(np.unique(m)) <= {0, 1} and rc == int(m.sum())
    return m


def changed_tiles(a, b, dw, dh):
    """Tiles of the coded picture whose oracle output differs between frames a and b."""
    cw, ch = r16(dw), r16(dh)
    ya, uva = oracle.csc_nv12(a, dw, dh, cw, ch)
    yb, uvb = oracle.csc_nv12(b, dw, dh, cw, ch)
    t = np.zeros((ch // 16, cw // 16), bool)
    yy, xx = np.nonzero(ya != yb)
    t[yy // 16, xx // 16] = True
    yy, xx = np.nonzero(uva != uvb)
    t[(2 * yy) // 16, xx // 16] = True
    return t


def random_rects(rng, sw, sh, n, min_size=1):
    out = []
    for _ in range(n):
        w, h = int(rng.integers(min_size, max(min_size + 1, sw // 3))), int(rng.integers(min_size, max(min_size + 1, sh // 3)))
        out.append((int(rng.integers(-w // 2, sw)), int(rng.integers(-h // 2, sh)), w, h))
    return out


def paint(rng, frame, rects):
    b = frame.copy()
    h, w = b.shape[:2]
    for x, y, rw, rh in rects:
        x0, y0, x1, y1 = max(x, 0), max(y, 0), min(x + rw, w), min(y + rh, h)
        if x1 > x0 and y1 > y0:
            b[y0:y1, x0:x1] = rng.integers(0, 256, (y1 - y0, x1 - x0, 4), dtype=np.uint8)
    return b


# (src, dst): 1:1 (even and odd-cropped), down and up both ways, and mixed
SIZES = [((64, 48), (64, 48)), ((1000, 562), (1000, 562)), ((250, 142), (250, 142)), ((320, 180), (160, 90)),
         ((1000, 562), (640, 360)), ((130, 98), (402, 306)), ((200, 120), (96, 250)), ((96, 64), (88, 72))]


@pytest.mark.parametrize("src,dst", SIZES)
def test_every_changed_sample_lies_in_a_dirty_tile(src, dst):
    rng = np.random.default_rng(hash((src, dst)) & 0xffff)
    (sw, sh), (dw, dh) = src, dst
    a = rng.integers(0, 256, (sh, sw, 4), dtype=np.uint8)
    for trial in range(4):
        rects = random_rects(rng, sw, sh, int(rng.integers(1, 6)))
        b = paint(rng, a, rects)
        m = tiles(sw, sh, dw, dh, rects)
        ch = changed_tiles(a, b, dw, dh)
        assert ch.shape == m.shape
        assert not (ch & (m == 0)).any(), f"{src}->{dst} rects {rects}: a changed tile is not dirty"


@pytest.mark.parametrize("size", [(64, 48), (1000, 562), (250, 142)])
def test_one_to_one_marks_exactly_the_tiles_a_rectangle_meets(size):
    rng = np.random.default_rng(7)
    sw, sh = size
    for trial in range(20):
        rects = random_rects(rng, sw, sh, int(rng.integers(0, 8)))
        want = np.zeros(((sh + 15) // 16, (sw + 15) // 16), np.uint8)
        for x, y, w, h in rects:
            x0, y0, x1, y1 = max(x, 0), max(y, 0), min(x + w, sw), min(y + h, sh)
            if x1 > x0 and y1 > y0:
                want[y0 // 16:(y1 - 1) // 16 + 1, x0 // 16:(x1 - 1) // 16 + 1] = 1
        assert np.array_equal(tiles(sw, sh, sw, sh, rects), want), rects


@pytest.mark.parametrize("src,dst", [s for s in SIZES if s[0] != s[1]])
def test_scaled_dirty_tiles_are_near_a_changed_tile(src, dst):
    rng = np.random.default_rng(11)
    (sw, sh), (dw, dh) = src, dst
    a = rng.integers(0, 256, (sh, sw, 4), dtype=np.uint8)
    for trial in range(4):
        rects = random_rects(rng, sw, sh, int(rng.integers(1, 4)), min_size=4)
        b = paint(rng, a, rects)
        m = tiles(sw, sh, dw, dh, rects).astype(bool)
        ch = changed_tiles(a, b, dw, dh)
        near = ch.copy()                  # every tile within one tile (8-neighbourhood) of a changed one
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                near |= np.roll(np.roll(ch, dy, 0), dx, 1) & ~_wrap(ch.shape, dy, dx)
        assert not (m & ~near).any(), f"{src}->{dst} rects {rects}: a dirty tile is more than one tile from any change"


def _wrap(shape, dy, dx):
    """The cells np.roll filled from the opposite edge."""
    w = np.zeros(shape, bool)
    if dy == 1:
        w[0] = True
    if dy == -1:
        w[-1] = True
    if dx == 1:
        w[:, 0] = True
    if dx == -1:
        w[:, -1] = True
    return w


def test_damage_tiles_edge_cases():
    assert not tiles(64, 48, 64, 48, []).any()
    assert not tiles(64, 48, 64, 48, [(64, 0, 10, 10), (0, 48, 5, 5), (-20, -20, 20, 20), (3, 3, 0, 9)]).any()
    assert tiles(64, 48, 64, 48, [(-5, -5, 1000, 1000)]).all()
    m = tiles(40, 34, 40, 34, [(39, 33, 1, 1)])            # the last pixel: its tile holds the padding of a cropped picture
    assert m.shape == (3, 3) and m[2, 2] == 1 and m.sum() == 1


def test_argument_errors_before_any_cuda_call():
    lib = N.lib()
    good, _ = N.rect_array([(0, 0, 4, 4)])
    many, n_many = N.rect_array([(0, 0, 1, 1)] * (N.B2V_MAX_DAMAGE_RECTS + 1))
    neg, _ = N.rect_array([(0, 0, 4, 4), (1, 1, -1, 2)])
    neg_h, _ = N.rect_array([(0, 0, 4, -3)])
    t = N.B2VTensor(0x1000, N.B2V_DT_U8, N.B2V_PIX_RGB, 1, 30, 3)
    calls = [lambda r, n: lib.b2v_ring_submit_damage(None, 0, 0, r, n, 0),
             lambda r, n: lib.b2v_submit_device_damage(None, 0x1000, 1280, N.B2V_PIX_BGRA, r, n, None, 0),
             lambda r, n: lib.b2v_submit_tensor_damage(None, t, r, n, None, 0)]
    for call in calls:
        assert call(many, n_many) == N.B2V_EINVAL and b"B2V_MAX_DAMAGE_RECTS" in lib.b2v_last_error()
        assert call(good, -1) == N.B2V_EINVAL and b"B2V_MAX_DAMAGE_RECTS" in lib.b2v_last_error()
        assert call(neg, 2) == N.B2V_EINVAL and b"negative" in lib.b2v_last_error()
        assert call(neg_h, 1) == N.B2V_EINVAL and b"negative" in lib.b2v_last_error()
        assert call(good, 1) == N.B2V_EINVAL and b"null handle" in lib.b2v_last_error()
        assert call(None, 0) == N.B2V_EINVAL and b"null" in lib.b2v_last_error()        # whole frame, null handle
    m = np.zeros(16, np.uint8)
    assert lib.b2v_damage_tiles(64, 64, 64, 64, many, n_many, m.ctypes.data) == N.B2V_EINVAL
    assert lib.b2v_damage_tiles(64, 64, 64, 64, neg, 2, m.ctypes.data) == N.B2V_EINVAL
    assert lib.b2v_damage_tiles(64, 64, 64, 64, good, 1, None) == N.B2V_EINVAL
    assert lib.b2v_damage_tiles(15, 64, 64, 64, good, 1, m.ctypes.data) == N.B2V_EINVAL
    assert lib.b2v_damage_tiles(64, 64, 64, 64, good, 1, m.ctypes.data) == 1


def test_rectangle_normalisation():
    assert normalize_rects([(-4, -4, 10, 10), (60, 30, 10, 10), (5, 5, 0, 3), (70, 0, 5, 5)], 64, 40) == [(0, 0, 6, 6), (60, 30, 4, 10)]
    with pytest.raises(ValueError):
        normalize_rects([(0, 0, -1, 4)], 64, 40)
    rng = np.random.default_rng(3)
    rects = [(int(rng.integers(0, 600)), int(rng.integers(0, 400)), int(rng.integers(1, 40)), int(rng.integers(1, 40))) for _ in range(300)]
    out = normalize_rects(rects, 640, 480)
    assert len(out) == N.B2V_MAX_DAMAGE_RECTS
    covered = np.zeros((480, 640), bool)
    for x, y, w, h in out:
        assert 0 <= x and 0 <= y and x + w <= 640 and y + h <= 480 and w > 0 and h > 0
        covered[y:y + h, x:x + w] = True
    for x, y, w, h in rects:
        assert covered[y:y + h, x:x + w].all()
    assert len(normalize_rects(rects[:N.B2V_MAX_DAMAGE_RECTS], 640, 480)) == N.B2V_MAX_DAMAGE_RECTS      # at the cap: kept as they are


class _Source(DamageFrameSource):
    def __init__(self, n):
        self.n, self.calls = n, []

    def fill_damage(self, view, index, whole):
        self.calls.append((index, whole))
        return None if index >= self.n else [(0, 0, 2, 2)]


class _Session:
    def __init__(self, refuse=()):
        self.calls, self.refuse = [], set(refuse)

    def acquire(self):
        return len(self.calls), np.zeros((4, 8, 4), np.uint8)

    def release_slot(self, slot):
        self.calls.append(("release", slot))

    def submit_slot(self, slot, capture_ns=0, damage=None):
        if damage is not None and slot in self.refuse:
            raise N.B2VError(N.B2V_ESTATE, "needs a whole picture")
        self.calls.append(("submit", slot, damage))

    def set_resolution(self, w, h):
        self.calls.append(("resize", w, h))


def test_screen_capture_asks_for_whole_frames_when_the_session_needs_them():
    src = _Source(5)
    cs = ScreenCapture(src)
    fake = _Session(refuse={2})
    assert all(cs._encode_next(fake, i) for i in range(3))
    cs._session = fake
    cs.update_resolution(8, 4)
    assert cs._encode_next(fake, 3) and cs._encode_next(fake, 4) and not cs._encode_next(fake, 5)
    # whole first; damage; refused -> the same slot filled whole and submitted whole; whole after the resize; damage; end
    assert src.calls == [(0, True), (1, False), (2, False), (2, True), (3, True), (4, False), (5, False)]
    assert fake.calls == [("submit", 0, None), ("submit", 1, [(0, 0, 2, 2)]), ("submit", 2, None), ("resize", 8, 4),
                          ("submit", 4, None), ("submit", 5, [(0, 0, 2, 2)]), ("release", 6)]


def test_screen_capture_fills_whole_past_the_cap():
    class Many(_Source):
        def fill_damage(self, view, index, whole):
            self.calls.append((index, whole))
            return [(i, 0, 1, 1) for i in range(N.B2V_MAX_DAMAGE_RECTS + 1)]
    src, fake = Many(9), _Session()
    cs = ScreenCapture(src)
    assert cs._encode_next(fake, 0) and cs._encode_next(fake, 1)
    assert src.calls == [(0, True), (1, False), (1, True)] and [c[2] for c in fake.calls] == [None, None]
