"""The picture size cap on the GPU (B2V_FLAG_SIZE_CAP): every access unit and reconstruction equal to the oracle's with the flag on,
through the two-sided driver (tests/cap_scenario.py mirrors the flag and the cap onto the oracle), which also decodes the GPU's own
stream.  Scroll restarts and video starts at 1080p and 4K, CQP and CBR, wide motion, droppable pictures, the long-term reference,
scene cuts, the quality flag, scaling, a resize, damage, device and tensor submits, a cap changed between pictures, and the contents on
which a recode changes macroblock kinds; striped mode against the independent model; the refusals and the three extra launches per
P picture."""
import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import cap_scenario as CS
from tests import device_scenario as D
from tests import scenario as S
from tests import tensor_scenario as T
from tests import h264_syntax_refs as HSR
from tests.test_size_cap_oracle import kinds_contents, scroll_restart, video_start

pytestmark = pytest.mark.gpu

CAP = N.B2V_FLAG_SIZE_CAP
assert CAP == CS.FLAG_SIZE_CAP


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


def _events(frames, cap):
    return [CS.set_max_picture_bytes(cap)] + S.stream(frames)


def _qps(segs):
    return [x.qp for x in S.pictures(segs)]


@pytest.mark.parametrize("extra", [0, N.B2V_FLAG_WIDE_MOTION | N.B2V_FLAG_LONG_TERM_REF | N.B2V_FLAG_SCENE_CUT | N.B2V_FLAG_QUALITY,
                                   N.B2V_FLAG_DROPPABLE | N.B2V_FLAG_WIDE_MOTION])
def test_contents_1080p(extra):
    w, h = 1920, 1080
    qps = []
    for frames in (scroll_restart(w, h), video_start(w, h)):
        qps += _qps(CS.run(S.Config(w, h, qp=24, flags=CAP | extra), _events(frames, 8000)))
    assert max(qps) > 24            # something was recoded


def test_4k_cbr():
    w, h = 3840, 2160
    frames = scroll_restart(w, h)[:5] + video_start(w, h)[2:4]
    CS.run(S.Config(w, h, rc_mode=S.CBR, kbps=20000, flags=CAP), _events(frames, 60000))


def test_live_cap_applies_from_the_next_picture():
    w, h = 640, 368
    frames = video_start(w, h)
    ev = S.stream(frames[:3]) + [CS.set_max_picture_bytes(2000)] + S.stream(frames[3:]) + [CS.set_max_picture_bytes(0)] + S.stream(frames)
    segs = CS.run(S.Config(w, h, qp=20, flags=CAP), ev)
    q = _qps(segs)
    assert q[:3] == [20] * 3 and max(q[3:6]) > 20


def test_cbr_paintover_scaling_resize_and_cropped():
    a, b = scroll_restart(1280, 720), video_start(800, 464)
    CS.run(S.Config(1280, 720, dst_width=960, dst_height=544, rc_mode=S.CBR, kbps=3000, paint=(2, 18, 2), flags=CAP),
           _events(a + [a[0]] * 3, 8000))
    CS.run(S.Config(1280, 720, qp=24, flags=CAP), _events(a, 10000) + [S.resize(800, 464)] + S.stream(b))
    CS.run(S.Config(330, 202, qp=18, flags=CAP), _events(video_start(330, 202), 3000))


def test_damage_device_and_tensor_frames():
    w, h = 640, 368
    with CS.oracle_side():
        D.run(D.DeviceConfig(w, h, qp=22, flags=CAP, pixel_format="RGBA", margin=(8, 4)), _events(video_start(w, h), 4000))
        T.run(T.TensorConfig(320, 192, qp=22, flags=CAP | N.B2V_FLAG_WIDE_MOTION, dtype="f16"), _events(video_start(320, 192), 2000))
    CS.run(S.Config(w, h, qp=22, flags=CAP | N.B2V_FLAG_DAMAGE), _events(scroll_restart(w, h), 3000))


def test_kinds_contents_parity():
    """The contents on which a recode turns coded macroblocks into P_Skip and back and I_PCM macroblocks into coded ones
    (tests/test_size_cap_oracle.py kinds_contents), bit-exact against the oracle."""
    for name, frames, qp, cap in kinds_contents(640, 368):
        segs = CS.run(S.Config(640, 368, qp=qp, flags=CAP), _events(frames, cap))
        assert _qps(segs)[1] > qp, name


def _striped(frames, cap, qp=20, stripe_rows=8):
    w, h = frames[0].shape[1], frames[0].shape[0]
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=qp, stripe_rows=stripe_rows, flags=CAP, max_picture_bytes=cap) as s:
        for f in frames:
            s.submit(f)
        s.flush()
        return s.take_frames()


def test_striped_decisions_follow_the_model():
    """Striped mode, where the cap applies to the whole access unit: from the flag-off stream (cap 0), the independent reader counts
    every picture over all its bands and the rule names the first recoded picture and its QP'; the capped stream is byte-identical up
    to it, codes every band of it at that QP', and every band's stream decodes."""
    from oracle import avdec
    from tests import h264_model_size_cap as M
    w, h, qp = 640, 368, 20
    frames = video_start(w, h)
    off, on = _striped(frames, 0, qp), _striped(frames, 3000, qp)

    def by_picture(got):
        bands, pics = {}, {}
        for x in got:
            bands.setdefault(x.y_start, []).append(x)
        for xs in bands.values():
            assert len(avdec.decode_stream([x.data for x in xs], quiet=True)) == len(xs)
            for x, pic in zip(xs, HSR.parse_stream([x.data for x in xs])):
                pics.setdefault(x.frame_id, []).append((x, pic))
        return [pics.get(k, []) for k in range(len(frames))]      # a picture whose every band is skipped delivers nothing

    a, b = by_picture(off), by_picture(on)
    first = None
    for k, (pa, pb) in enumerate(zip(a, b)):
        if k == 0:
            continue
        bits = sum(M.count(pic) for _, pic in pa)
        want = M.qp_after(bits, qp, 3000)
        if want != qp:
            first = k
            assert {x.qp for x, _ in pb} == {want} and {pic.qp for _, pic in pb} == {want}, (k, want)
            break
        assert [x.data for x, _ in pa] == [x.data for x, _ in pb], k
    assert first is not None


def _launches(cap, frames):
    with Session(320, 192, rc_mode=N.B2V_RC_CQP, crf=26, flags=CAP if cap else 0) as s:
        for f in frames:
            s.submit(f)
        s.flush()
        return len(s.take_frames()), s.stats()["kernel_launches"]


def test_kernel_launches():
    """Three more launches per P picture with the flag (k_size_cap, k_requant, the second CAVLC pass), none for the IDR picture."""
    frames = video_start(320, 192)
    n, off = _launches(False, frames)
    n2, on = _launches(True, frames)
    assert n == n2 == len(frames) and on == off + 3 * (len(frames) - 1)


def test_refusals():
    for kw in (dict(flags=N.B2V_FLAG_JPEG), dict(flags=N.B2V_FLAG_NO_ENCODE)):
        with pytest.raises(N.B2VError) as e:
            Session(320, 256, max_picture_bytes=1000, **kw)
        assert e.value.code == N.B2V_EINVAL and "SIZE_CAP" in str(e.value), kw
    with Session(320, 256) as s:
        with pytest.raises(N.B2VError) as e:
            s.set_max_picture_bytes(1000)
        assert e.value.code == N.B2V_ESTATE
    with Session(320, 256, flags=CAP) as s:
        with pytest.raises(N.B2VError) as e:
            s.set_max_picture_bytes(-1)
        assert e.value.code == N.B2V_EINVAL
        s.set_max_picture_bytes(0)
    with pytest.raises(N.B2VError) as e:
        Session(320, 256, max_picture_bytes=-5)
    assert e.value.code == N.B2V_EINVAL
