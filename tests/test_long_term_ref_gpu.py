"""The long-term reference picture on the GPU (B2V_FLAG_LONG_TERM_REF): every access unit and reconstruction equal to the oracle's with
the flag on, through the two-sided driver (tests/ltr_scenario.py mirrors the flag onto the oracle), which also decodes the GPU's own
stream to its reconstructions.  Covers the scripted contents of tests/ltr_content.py at 1080p, CQP and CBR with an IDR request and a
gop, paint-over, scaling and a resize, a cropped odd size, wide-range motion, the quality flag and the 4K headline configuration;
also the refusals and the one extra launch per P picture."""
import dataclasses

import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import ltr_content as LC
from tests import ltr_scenario as LS
from tests import scenario as S
from tests import synth

pytestmark = pytest.mark.gpu

LTR = N.B2V_FLAG_LONG_TERM_REF
assert LTR == LS.FLAG_LONG_TERM_REF


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


@pytest.mark.parametrize("name", sorted(LC.CONTENTS))
def test_contents_1080p(name):
    w, h = 1920, 1080
    frames, _ = LC.CONTENTS[name](w, h)
    LS.run(S.Config(w, h, qp=26, flags=LTR), S.stream(frames))


def test_wide_motion_and_quality():
    w, h = 1920, 1080
    frames = LC.alt_tab(w, h)[0] + LC.drag(w, h)[0]
    LS.run(S.Config(w, h, qp=28, flags=LTR | N.B2V_FLAG_WIDE_MOTION | N.B2V_FLAG_QUALITY), S.stream(frames))


def test_cbr_idr_request_gop_and_paintover():
    w, h = 1280, 720
    frames = LC.popup(w, h)[0] + LC.alt_tab(w, h)[0]
    ev = S.stream(frames[:8]) + [S.request_idr()] + S.stream(frames[8:14]) + [S.set_gop(5)] + S.stream(frames[14:])
    LS.run(S.Config(w, h, rc_mode=S.CBR, kbps=6000, paint=(3, 18, 2), flags=LTR), ev)


def test_scaled_resize_and_cropped():
    LS.run(S.Config(1280, 720, dst_width=960, dst_height=544, qp=30, flags=LTR), S.stream(LC.popup(1280, 720)[0]))
    a, b = LC.alt_tab(640, 368)[0], LC.popup(800, 464)[0]
    LS.run(S.Config(640, 368, qp=28, flags=LTR), S.stream(a) + [S.resize(800, 464)] + S.stream(b))
    LS.run(S.Config(330, 202, qp=24, flags=LTR), S.stream(LC.popup(330, 202)[0]))


def test_headline_4k():
    """bench.py's configuration (4K, CBR 20 Mbit/s, resident frames) with the flag, on its own contents and on an app switch."""
    from tests.test_inter_passes_gpu import BENCH, N_DISTINCT, W, H
    frames = [synth.desktop(W, H, t) for t in range(N_DISTINCT)]
    cfg = dataclasses.replace(BENCH, flags=BENCH.flags | LTR)
    LS.run(cfg, [S.picture(frames[i % N_DISTINCT]) for i in range(34)])
    LS.run(cfg, S.stream(LC.alt_tab(W, H)[0]))


def _launches(ltr, frames, **kw):
    with Session(320, 192, rc_mode=N.B2V_RC_CQP, crf=26, long_term_ref=ltr, **kw) as s:
        for f in frames:
            s.submit(f)
        s.flush()
        return len(s.take_frames()), s.stats()["kernel_launches"]


def test_kernel_launches():
    """One more launch per P picture with the flag (k_ltr_mark), none for the IDR picture; none without the flag."""
    frames = LC.popup(320, 192)[0]
    n, off = _launches(False, frames)
    n2, on = _launches(True, frames)
    assert n == n2 == len(frames) and on == off + len(frames) - 1


def test_create_refusals():
    cases = (dict(flags=N.B2V_FLAG_JPEG), dict(flags=N.B2V_FLAG_NO_ENCODE), dict(droppable=True), dict(stripe_rows=4))
    for kw in cases:
        with pytest.raises(N.B2VError) as e:
            Session(320, 256, long_term_ref=True, **kw)
        assert e.value.code == N.B2V_EINVAL, kw
        assert "LONG_TERM_REF" in str(e.value), kw


def test_resize_that_would_stripe_is_refused():
    with Session(320, 64, stripe_rows=4, long_term_ref=True) as s:
        with pytest.raises(N.B2VError) as e:
            s.set_resolution(320, 256)
        assert e.value.code == N.B2V_EINVAL and "LONG_TERM_REF" in str(e.value)
