"""Droppable pictures on the GPU (B2V_FLAG_DROPPABLE): every access unit and reconstruction equal to the oracle's with the flag on,
through the two-sided driver (tests/layered_scenario.py mirrors the flag onto the oracle's LayeredRefEncoder), across CQP, CBR with IDR requests
and a gop, scaling, a resize, the 4K headline configuration, every exit of the motion search, device and tensor frames, together
with B2V_FLAG_QUALITY and over a frame_num wrap; the GPU's own stream without its non-reference access units decodes to the GPU's
reconstructions; and the combinations b2v_create refuses."""
import dataclasses

import numpy as np
import pytest

import oracle
from oracle import avdec
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import device_scenario as D
from tests import layered_scenario as LS
from tests import scenario as S
from tests import synth
from tests import tensor_scenario as T

pytestmark = pytest.mark.gpu

DROP = N.B2V_FLAG_DROPPABLE
assert DROP == LS.FLAG_DROPPABLE


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


def desktop(w, h, n, t0=0):
    return [synth.desktop(w, h, t0 + t) for t in range(n)]


def _layers(xs):
    """nal_ref_idc of each picture's first slice NAL, from the oracle's access units (equal to the GPU's by the comparison)."""
    out = []
    for x in xs:
        au = x.au
        i = 0
        while True:
            i = au.find(b"\x00\x00\x01", i) + 3
            if au[i] & 31 in (1, 5):
                out.append(au[i] >> 5 & 3)
                break
    return out


@pytest.mark.parametrize("qp", [0, 26, 51])
def test_cqp(qp):
    w, h = 640, 368
    xs = S.pictures(LS.run(S.Config(w, h, qp=qp, flags=DROP), S.stream(desktop(w, h, 9))))
    assert _layers(xs) == [3] + [0, 2] * 4


def test_cbr_idr_request_and_gop():
    w, h = 1280, 720
    frames = desktop(w, h, 24)
    ev = S.stream(frames[:5]) + [S.request_idr()] + S.stream(frames[5:12]) + [S.set_gop(4)] + S.stream(frames[12:])
    xs = S.pictures(LS.run(S.Config(w, h, rc_mode=S.CBR, kbps=6000, flags=DROP), ev))
    keys = [k for k, x in enumerate(xs) if x.is_key]
    assert keys[:2] == [0, 5] and len(keys) >= 4
    layers = _layers(xs)
    since = 0
    for k, x in enumerate(xs):
        since = 0 if x.is_key else since + 1
        assert layers[k] == (3 if x.is_key else 0 if since % 2 else 2), (k, layers)


def test_scaled():
    LS.run(S.Config(1280, 720, dst_width=960, dst_height=544, qp=30, flags=DROP), S.stream(desktop(1280, 720, 8)))


def test_resize_mid_stream():
    a, b = desktop(640, 368, 5), desktop(800, 464, 6)
    LS.run(S.Config(640, 368, qp=28, flags=DROP), S.stream(a) + [S.resize(800, 464)] + S.stream(b))


def test_headline_4k_two_scroll_restarts():
    """bench.py's configuration (4K, CBR 20 Mbit/s, resident frames) with the flag, across the scroll restarts at 16 and 32."""
    from tests.test_inter_passes_gpu import BENCH, N_DISTINCT, W, H
    frames = desktop(W, H, N_DISTINCT)
    cfg = dataclasses.replace(BENCH, flags=BENCH.flags | DROP)
    xs = S.pictures(LS.run(cfg, [S.picture(frames[i % N_DISTINCT]) for i in range(34)]))
    assert _layers(xs) == [3] + [0, 2] * 16 + [0]


def test_predictor_paths():
    w, h = 640, 368
    LS.run(S.Config(w, h, qp=30, flags=DROP), S.stream(synth.predictor_paths(w, h)))


def test_device_frames():
    w, h = 640, 368
    with LS.oracle_side():
        D.run(D.DeviceConfig(w, h, qp=27, flags=DROP, pixel_format="RGBA", margin=(8, 4)), S.stream(desktop(w, h, 7)))


def test_tensor_frames():
    w, h = 320, 192
    cfg = T.TensorConfig(w, h, qp=26, flags=DROP, dtype="f16")
    with LS.oracle_side():
        T.run(cfg, S.stream(desktop(w, h, 7)))


def test_with_quality_flag():
    w, h = 640, 368
    LS.run(S.Config(w, h, qp=26, flags=DROP | N.B2V_FLAG_QUALITY), S.stream(desktop(w, h, 7)))


def test_frame_num_wraps():
    """530 pictures: 265 reference pictures, so frame_num (8 bits, advancing after reference pictures only) wraps once."""
    w, h = 160, 96
    frames = desktop(w, h, 24)
    xs = S.pictures(LS.run(S.Config(w, h, qp=30, flags=DROP, ring_slots=8), [S.picture(frames[i % 24]) for i in range(530)]))
    assert sum(1 for v in _layers(xs) if v) > 256


def test_reference_substream_of_the_gpu_decodes_to_its_reconstructions():
    """The GPU's own access units, picture by picture with its reconstruction after each: the stream without every non-reference
    access unit decodes to the reconstructions of the pictures kept, and the whole stream to all of them."""
    w, h = 640, 368
    aus, recs = [], []
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=26, droppable=True) as s:
        for f in desktop(w, h, 11):
            s.submit(f)
            recs.append(s.recon())
            fr, = s.take_frames()
            aus.append(fr)
    assert [f.droppable for f in aus] == [False] + [k % 2 == 1 for k in range(1, 11)]
    for keep in (range(len(aus)), [k for k, f in enumerate(aus) if not f.droppable]):
        dec = avdec.decode_stream([aus[k].data for k in keep], quiet=True)
        assert len(dec) == len(keep)
        for (Y, U, V), k in zip(dec, keep):
            y, uv = recs[k]
            assert np.array_equal(Y, y[:h, :w]) and np.array_equal(U, uv[:h // 2, 0:w:2]) and np.array_equal(V, uv[:h // 2, 1:w:2]), k


def test_pixelflux_header_marks_droppable_frames():
    w, h = 320, 192
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=26, header_mode=N.B2V_HDR_PIXELFLUX, droppable=True) as s:
        for f in desktop(w, h, 5):
            s.submit(f)
        s.flush()
        got = s.take_frames()
    assert [f.droppable for f in got] == [False, True, False, True, False]
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=26) as s:
        for f in desktop(w, h, 3):
            s.submit(f)
        s.flush()
        assert not any(f.droppable for f in s.take_frames())


def test_create_refusals():
    for kw in (dict(flags=N.B2V_FLAG_JPEG), dict(flags=N.B2V_FLAG_NO_ENCODE), dict(stripe_rows=4)):
        with pytest.raises(N.B2VError) as e:
            Session(320, 256, droppable=True, **kw)
        assert e.value.code == N.B2V_EINVAL, kw
        assert "DROPPABLE" in str(e.value), kw
    # stripe_rows >= the picture's rows is full frame: allowed; a resize to a size it would stripe is refused
    with Session(320, 64, stripe_rows=4, droppable=True) as s:
        with pytest.raises(N.B2VError) as e:
            s.set_resolution(320, 256)
        assert e.value.code == N.B2V_EINVAL
        s.submit(synth.desktop(320, 64, 0))
        s.flush()
        assert len(s.take_frames()) == 1
