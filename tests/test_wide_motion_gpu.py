"""Wide-range motion on the GPU (B2V_FLAG_WIDE_MOTION): every access unit and reconstruction equal to the oracle's with the flag on,
through the two-sided driver (tests/wide_scenario.py mirrors the flag onto the oracle), which also decodes the GPU's own stream to its
reconstructions.  Covers CQP 0/26/51, CBR with an IDR request and a gop, scaling and a resize, bands that clamp the coarse search,
droppable pictures, the quality flag, device and tensor frames, pictures smaller than one anchor group, a cropped odd size, the 4K
headline configuration, and a steady fast scroll whose wide vectors the temporal predictor carries through k_inter_lean; also the
refusals and the kernel launches."""
import dataclasses

import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import device_scenario as D
from tests import scenario as S
from tests import synth
from tests import tensor_scenario as T
from tests import wide_content as WC
from tests import wide_scenario as WS

pytestmark = pytest.mark.gpu

WIDE = N.B2V_FLAG_WIDE_MOTION
assert WIDE == WS.FLAG_WIDE_MOTION


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


def scroll(w, h, speed, n, still=1):
    """`still` copies of the first picture, then the scroll: the motion starts inside the stream."""
    return [WC.desktop_scroll(w, h, 0, speed)] * still + [WC.desktop_scroll(w, h, t, speed) for t in range(1, n - still + 1)]


@pytest.mark.parametrize("qp", [0, 26, 51])
def test_cqp(qp):
    w, h = 640, 368
    WS.run(S.Config(w, h, qp=qp, flags=WIDE), S.stream(scroll(w, h, 40, 7)))


def test_cbr_idr_request_and_gop():
    w, h = 1280, 720
    frames = scroll(w, h, 64, 20)
    ev = S.stream(frames[:5]) + [S.request_idr()] + S.stream(frames[5:11]) + [S.set_gop(4)] + S.stream(frames[11:])
    WS.run(S.Config(w, h, rc_mode=S.CBR, kbps=6000, flags=WIDE), ev)


def test_scaled_and_resize():
    WS.run(S.Config(1280, 720, dst_width=960, dst_height=544, qp=30, flags=WIDE), S.stream(scroll(1280, 720, 48, 7)))
    a, b = scroll(640, 368, 24, 5), scroll(800, 464, 100, 6)
    WS.run(S.Config(640, 368, qp=28, flags=WIDE), S.stream(a) + [S.resize(800, 464)] + S.stream(b))


@pytest.mark.parametrize("rows", [2, 5])
def test_striped_bands_clamp_the_coarse_search(rows):
    w, h = 640, 480
    WS.run(S.Config(w, h, qp=27, stripe_rows=rows, flags=WIDE), S.stream(scroll(w, h, 40, 7)))


def test_droppable():
    w, h = 1280, 720
    WS.run(S.Config(w, h, qp=26, flags=WIDE | N.B2V_FLAG_DROPPABLE), S.stream(scroll(w, h, 128, 10)))


def test_with_quality_flag():
    w, h = 640, 368
    WS.run(S.Config(w, h, qp=26, flags=WIDE | N.B2V_FLAG_QUALITY), S.stream(scroll(w, h, 40, 6)))


def test_drags_and_existing_contents():
    w, h = 1280, 720
    for v in [(40, -30), (-100, 0), (127, 60)]:
        start = (560 - 2 * v[0], 240 - 2 * v[1])
        WS.run(S.Config(w, h, qp=26, flags=WIDE), S.stream([WC.drag(w, h, 0, v, start)] + [WC.drag(w, h, t, v, start) for t in range(5)]))
    WS.run(S.Config(640, 368, qp=30, flags=WIDE), S.stream(synth.predictor_paths(640, 368)))


def test_device_frames():
    w, h = 640, 368
    with WS.oracle_side():
        D.run(D.DeviceConfig(w, h, qp=27, flags=WIDE, pixel_format="RGBA", margin=(8, 4)), S.stream(scroll(w, h, 40, 7)))


def test_tensor_frames():
    w, h = 320, 192
    with WS.oracle_side():
        T.run(T.TensorConfig(w, h, qp=26, flags=WIDE, dtype="f16"), S.stream(scroll(w, h, 24, 7)))


@pytest.mark.parametrize("size", [(16, 16), (48, 32), (330, 202)])
def test_small_and_cropped_sizes(size):
    """16x16 and 48x32: the decimated plane is smaller than one anchor group; 330x202: cropped, edge groups of one macroblock."""
    w, h = size
    WS.run(S.Config(w, h, qp=24, flags=WIDE), S.stream([WC.drag(w, h, t, (-7, 5), (w // 3, h // 4), max(8, w // 2), max(8, h // 2)) for t in range(6)]))


def test_headline_4k():
    """bench.py's configuration (4K, CBR 20 Mbit/s, resident frames) with the flag, across the scroll restarts at 16 and 32."""
    from tests.test_inter_passes_gpu import BENCH, N_DISTINCT, W, H
    frames = [synth.desktop(W, H, t) for t in range(N_DISTINCT)]
    WS.run(dataclasses.replace(BENCH, flags=BENCH.flags | WIDE), [S.picture(frames[i % N_DISTINCT]) for i in range(34)])


def test_steady_fast_scroll_through_the_lean_pass():
    """A 1080p scroll of 96 px per picture, long enough that the wide vector is the temporal predictor of every moving macroblock."""
    w, h = 1920, 1080
    WS.run(S.Config(w, h, qp=26, flags=WIDE), S.stream(scroll(w, h, 96, 12)))


def _launches(wide, frames, **kw):
    with Session(320, 192, rc_mode=N.B2V_RC_CQP, crf=26, wide_motion=wide, **kw) as s:
        for f in frames:
            s.submit(f)
        s.flush()
        return len(s.take_frames()), s.stats()["kernel_launches"]


def test_kernel_launches():
    """One more launch per picture with the flag (k_coarse), IDR pictures included; none without it."""
    frames = scroll(320, 192, 24, 6)
    n, off = _launches(False, frames)
    n2, on = _launches(True, frames)
    assert n == n2 == 6 and on == off + 6


def test_create_refusals():
    for kw in (dict(flags=N.B2V_FLAG_JPEG), dict(flags=N.B2V_FLAG_NO_ENCODE)):
        with pytest.raises(N.B2VError) as e:
            Session(320, 256, wide_motion=True, **kw)
        assert e.value.code == N.B2V_EINVAL, kw
        assert "WIDE_MOTION" in str(e.value), kw
