"""Scene cuts on the GPU (B2V_FLAG_SCENE_CUT): every access unit and reconstruction equal to the oracle's with the flag on, through the
two-sided driver (tests/scut_scenario.py mirrors the flag onto the oracle), which also decodes the GPU's own stream to its
reconstructions.  Covers whole-screen switches and the scripted contents of tests/ltr_content.py at 1080p and 4K, CQP and CBR with
an IDR request and a gop, paint-over, scaling and a resize, a cropped size, wide-range motion, droppable pictures, the long-term
reference, the quality flag, device and tensor submits; also EncodedFrame.intra, the refusals and the two extra launches per P
picture."""
import dataclasses

import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.h264_nal import is_intra
from selkies_b200.session import Session
from tests import device_scenario as D
from tests import ltr_content as LC
from tests import scenario as S
from tests import scut_scenario as SC
from tests import tensor_scenario as T

pytestmark = pytest.mark.gpu

CUT = N.B2V_FLAG_SCENE_CUT
assert CUT == SC.FLAG_SCENE_CUT


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


def _cuts(segs):
    return [k for k, x in enumerate(S.pictures(segs)) if is_intra(x.bands[0][1]) and not x.is_key]


@pytest.mark.parametrize("extra", [0, N.B2V_FLAG_WIDE_MOTION | N.B2V_FLAG_LONG_TERM_REF | N.B2V_FLAG_QUALITY,
                                   N.B2V_FLAG_DROPPABLE | N.B2V_FLAG_WIDE_MOTION])
def test_switches_1080p(extra):
    w, h = 1920, 1080
    segs = SC.run(S.Config(w, h, qp=26, flags=CUT | extra), S.stream(SC.switches(w, h)))
    cuts = _cuts(segs)
    # switches cut; stills and desktop -> desktop stay P.  With droppable pictures picture 6 (odd count) predicts from picture 4,
    # two back, for which its content is new.
    stills = {0, 1, 3, 9} | (set() if extra & N.B2V_FLAG_DROPPABLE else {6})
    assert 2 in cuts and 5 in cuts and not stills & set(cuts), cuts


@pytest.mark.parametrize("name", ["popup", "alt_tab", "drag", "scroll"])
def test_contents_1080p(name):
    w, h = 1920, 1080
    frames, _ = LC.CONTENTS[name](w, h)
    SC.run(S.Config(w, h, qp=36, flags=CUT | N.B2V_FLAG_LONG_TERM_REF), S.stream(frames))


def test_cbr_idr_request_gop_and_paintover():
    w, h = 1280, 720
    frames = SC.switches(w, h) + LC.alt_tab(w, h)[0]
    ev = S.stream(frames[:8]) + [S.request_idr()] + S.stream(frames[8:16]) + [S.set_gop(5)] + S.stream(frames[16:])
    SC.run(S.Config(w, h, rc_mode=S.CBR, kbps=6000, paint=(3, 18, 2), flags=CUT), ev)


def test_scaled_resize_and_cropped():
    SC.run(S.Config(1280, 720, dst_width=960, dst_height=544, qp=30, flags=CUT), S.stream(SC.switches(1280, 720)))
    a, b = SC.switches(640, 368), LC.alt_tab(800, 464)[0]
    SC.run(S.Config(640, 368, qp=28, flags=CUT | N.B2V_FLAG_DROPPABLE), S.stream(a) + [S.resize(800, 464)] + S.stream(b))
    SC.run(S.Config(330, 202, qp=24, flags=CUT), S.stream(SC.switches(330, 202)))


def test_device_and_tensor_frames():
    w, h = 640, 368
    with SC.oracle_side():
        D.run(D.DeviceConfig(w, h, qp=27, flags=CUT, pixel_format="RGBA", margin=(8, 4)), S.stream(SC.switches(w, h)))
        T.run(T.TensorConfig(320, 192, qp=26, flags=CUT | N.B2V_FLAG_WIDE_MOTION, dtype="f16"), S.stream(SC.switches(320, 192)))


def test_headline_4k():
    """bench.py's configuration (4K, CBR 20 Mbit/s, resident frames) with the flag, on whole-screen switches and an app switch."""
    from tests.test_inter_passes_gpu import BENCH, W, H
    cfg = dataclasses.replace(BENCH, flags=BENCH.flags | CUT)
    SC.run(cfg, S.stream(SC.switches(W, H)[:8]))
    SC.run(dataclasses.replace(cfg, flags=cfg.flags | N.B2V_FLAG_LONG_TERM_REF), S.stream(LC.alt_tab(W, H)[0]))


def test_encoded_frame_intra():
    """EncodedFrame.intra on exactly the cut pictures: the P pictures whose first slice is an I slice; never on an IDR."""
    w, h = 320, 192
    frames = SC.switches(w, h)
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=26, scene_cut=True) as s:
        for f in frames:
            s.submit(f)
        s.flush()
        got = s.take_frames()
    assert len(got) == len(frames) and got[0].is_key and not got[0].intra
    cuts = [k for k, x in enumerate(got) if x.intra]
    assert cuts and cuts == [k for k, x in enumerate(got) if not x.is_key and is_intra(x.data)]
    assert all(not x.is_key for x in got[1:])
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=26) as s:
        for f in frames:
            s.submit(f)
        s.flush()
        assert not any(x.intra for x in s.take_frames())


def _launches(cut, frames, **kw):
    with Session(320, 192, rc_mode=N.B2V_RC_CQP, crf=26, scene_cut=cut, **kw) as s:
        for f in frames:
            s.submit(f)
        s.flush()
        return len(s.take_frames()), s.stats()["kernel_launches"]


def test_kernel_launches():
    """Two more launches per P picture with the flag (k_scene_cut, k_intra_rows), none for the IDR picture; none without it."""
    frames = SC.switches(320, 192)
    n, off = _launches(False, frames)
    n2, on = _launches(True, frames)
    assert n == n2 == len(frames) and on == off + 2 * (len(frames) - 1)


def test_create_refusals():
    for kw in (dict(flags=N.B2V_FLAG_JPEG), dict(flags=N.B2V_FLAG_NO_ENCODE), dict(stripe_rows=4)):
        with pytest.raises(N.B2VError) as e:
            Session(320, 256, scene_cut=True, **kw)
        assert e.value.code == N.B2V_EINVAL, kw
        assert "SCENE_CUT" in str(e.value), kw


def test_resize_that_would_stripe_is_refused():
    with Session(320, 64, stripe_rows=4, scene_cut=True) as s:
        with pytest.raises(N.B2VError) as e:
            s.set_resolution(320, 256)
        assert e.value.code == N.B2V_EINVAL and "SCENE_CUT" in str(e.value)
