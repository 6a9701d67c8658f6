"""GPU: every stripe the JPEG mode delivers (B2V_FLAG_JPEG) against libjpeg-turbo directly, not through the oracle.

On grey pictures and on mosaics of agreeing colours (tests/jpeg_libjpeg.py) libjpeg-turbo's 4:2:0 file of the stripe's rows,
edge-padded to the coded size and with SOF saying the visible size, is what the library must deliver byte for byte.  This
reaches what the oracle parity of test_jpeg_gpu.py cannot tell apart from a mistake made the same way in both encoders: the
chroma quantiser and Huffman tables, the MCU interleave, the DC predictors and the clamps of the quality rule."""
import numpy as np
import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests.test_jpeg_gpu import stripe_rows_of

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
from tests import jpeg_libjpeg as J  # noqa: E402  (needs cv2)


@pytest.fixture(scope="module")
def palette():
    return J.agreeing_palette(np.random.default_rng(11), 2000)


def picture(kind, w, h, request, seed=1):
    if kind == "palette":                      # (grey cases do not depend on the palette fixture)
        return J.mosaic(request.getfixturevalue("palette"), w, h, seed)
    return J.grey_noise(w, h, seed) if w * h <= 130 * 70 else J.grey_desktop(w, h, seed)


def check_stripes(got, frame, quality, rows, frame_id=0):
    """`got`: the stripes of one picture in delivery order, every stripe of it delivered."""
    h, w = frame.shape[:2]
    assert [(g.y_start, g.height, g.frame_id) for g in got] == [(y0, min(rows, h - y0), frame_id) for y0 in range(0, h, rows)]
    for g in got:
        ref = J.stripe_reference(frame, g.y_start, rows, quality)
        assert g.data == ref, f"{w}x{h} stripe at row {g.y_start}, quality {quality}: {J.difference(g.data, ref, w)}"


def encode(w, h, frames, crf, stripe_rows=0, **kw):
    with Session(w, h, flags=N.B2V_FLAG_JPEG, rc_mode=N.B2V_RC_CQP, crf=crf, stripe_rows=stripe_rows, **kw) as s:
        for f in frames:
            s.submit(f)
            s.flush()
        return s.take_frames()


QUALITIES = [1, 19, 24, 50, 100, 0]          # 0: the default, 60


@pytest.mark.parametrize("kind", ["grey", "palette"])
@pytest.mark.parametrize("crf", QUALITIES)
@pytest.mark.parametrize("w,h,stripe_rows", [(16, 16, 1), (16, 16, 67), (130, 70, 1), (130, 70, 3), (130, 70, 5), (130, 70, 0),
                                             (1920, 1080, 0)])
def test_every_stripe_is_libjpeg_turbos_file(w, h, stripe_rows, crf, kind, request):
    """Qualities on both sides of the clamp to 255 (luma below 24, chroma below 20) and the clamp to 1 at 100; one-row
    stripes, stripes of 3 rows whose last one is short, a stripe of every row and the default rule; 1920x1080's last MCU row
    holds 8 visible rows."""
    f = picture(kind, w, h, request)
    check_stripes(encode(w, h, [f], crf, stripe_rows), f, crf or 60, stripe_rows_of(h, stripe_rows) * 16)


@pytest.mark.parametrize("w,h,stripe_rows,crf,kind", [(1920, 1080, 67, 19, "palette"), (1920, 1080, 68, 100, "grey"),
                                                      (3840, 2160, 0, 24, "palette"), (3840, 2160, 1, 100, "grey"),
                                                      (7680, 4320, 0, 1, "palette"), (7680, 4320, 3, 50, "grey")])
def test_large_pictures(w, h, stripe_rows, crf, kind, request):
    f = picture(kind, w, h, request)
    check_stripes(encode(w, h, [f], crf, stripe_rows), f, crf, stripe_rows_of(h, stripe_rows) * 16)


def test_densest_content_fits_at_4k():
    """Black / white grey noise at quality 100, about 81 B per block against an output capacity of 128: the access unit must
    not overflow (an overflowing one fails the session and delivers nothing), picture after picture."""
    w, h = 3840, 2160
    frames = [J.grey_noise(w, h, seed, binary=True) for seed in (1, 2)]
    got = encode(w, h, frames, 100)
    rows = stripe_rows_of(h, 0) * 16
    for k, f in enumerate(frames):
        check_stripes([g for g in got if g.frame_id == k], f, 100, rows, k)
    assert sum(len(g.data) for g in got) / (2 * w * h * 6 // 256) > 70


@pytest.mark.parametrize("crf,paint", [(1, 100), (100, 1)])
def test_paintover_stripes_carry_their_own_quality(crf, paint, palette):
    """Picture 1 repeats picture 0: every stripe is repainted at the paint-over quality.  Picture 2 changes stripe 2 only: it
    alone is sent, at the normal quality, and repainted in picture 3."""
    w, h, rows = 320, 192, 48
    a = J.mosaic(palette, w, h, 1)
    b = a.copy()
    b[100:110, 40:80] = J.mosaic(palette, 40, 10, 2)
    got = encode(w, h, [a, a, b, b], crf, 3, paintover_trigger_frames=1, paintover_crf=paint)
    by = {k: [g for g in got if g.frame_id == k] for k in range(4)}
    check_stripes(by[0], a, crf, rows, 0)
    check_stripes(by[1], a, paint, rows, 1)
    assert [g.y_start for g in by[2]] == [96] and by[2][0].data == J.stripe_reference(b, 96, rows, crf)
    assert [g.y_start for g in by[3]] == [96] and by[3][0].data == J.stripe_reference(b, 96, rows, paint)


@pytest.mark.parametrize("sw,sh,dw,dh", [(3840, 2160, 1920, 1080), (1920, 1080, 320, 180)])
def test_scaled_grey(sw, sh, dw, dh):
    """Scaled sessions through both shared-memory tiers of the tiled scale kernel.  A bilinear scale of greys is grey, so the
    stripes are libjpeg-turbo's files of the scaled luma plane."""
    f = J.grey_desktop(sw, sh, 2)
    y, uv = oracle.csc_nv12(f, dst_w=dw, dst_h=dh, matrix=1)
    assert (uv == 128).all()
    with Session(sw, sh, dst_width=dw, dst_height=dh, flags=N.B2V_FLAG_JPEG, rc_mode=N.B2V_RC_CQP, crf=50) as s:
        s.submit(f)
        s.flush()
        got = s.take_frames()
    check_stripes(got, J.grey(y), 50, stripe_rows_of(dh, 0) * 16)


def test_resize_mid_stream(palette):
    """set_resolution changes the stripe count and width; the first picture after it delivers every stripe."""
    sizes = [(320, 192), (130, 70), (1920, 1080)]
    pics = [J.mosaic(palette, w, h, k) for k, (w, h) in enumerate(sizes)]
    with Session(*sizes[0], flags=N.B2V_FLAG_JPEG, rc_mode=N.B2V_RC_CQP, crf=24, stripe_rows=2) as s:
        for k, ((w, h), f) in enumerate(zip(sizes, pics)):
            if k:
                s.set_resolution(w, h)
            s.submit(f)
            s.submit(f)                                    # unchanged: nothing to deliver
            s.flush()
            got = s.take_frames()
            ids = sorted({g.frame_id for g in got})
            assert len(ids) == 1, ids
            check_stripes(got, f, 24, 32, ids[0])


def test_device_and_tensor_sources(palette):
    """An RGB uint8 frame through submit_device and a grey CHW fp16 tensor through submit_tensor."""
    torch = pytest.importorskip("torch")
    from tests import tensor_scenario as T
    w, h = 640, 360
    f = J.mosaic(palette, w, h, 3)
    rgb = torch.from_numpy(np.ascontiguousarray(f[..., 2::-1])).cuda()
    with Session(w, h, flags=N.B2V_FLAG_JPEG, rc_mode=N.B2V_RC_CQP, crf=100) as s:
        s.submit_device(rgb, pixel_format="RGB")
        s.flush()
        check_stripes(s.take_frames(), f, 100, stripe_rows_of(h, 0) * 16)
    v = torch.rand(h, w, generator=torch.Generator().manual_seed(4)).half()
    g = J.grey(T.quantise(v.float().numpy()))
    with Session(w, h, flags=N.B2V_FLAG_JPEG, rc_mode=N.B2V_RC_CQP, crf=19) as s:
        s.submit_tensor(v.cuda().expand(3, h, w).contiguous(), channels="RGB", layout="CHW")
        s.flush()
        check_stripes(s.take_frames(), g, 19, stripe_rows_of(h, 0) * 16)
