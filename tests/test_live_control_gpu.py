"""GPU parity under live control (tests/scenario.py driver, scripts in tests/longrun_scripts.py): set_bitrate_kbps /
set_framerate / set_qp / set_gop / request_idr / set_resolution called between submits while pictures are in flight, as REMB
and PLI feedback, keyframe_distance and client resizes do in a session.  A call made after submit k applies from picture k+1
(include/b2video.h) on both sides; every access unit, QP, key flag and frame id must equal the oracle's."""
import numpy as np
import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import longrun_scripts as L
from tests import scenario as S
from tests import synth

pytestmark = pytest.mark.gpu


def test_cbr_bitrate_and_framerate_steps():
    L.check_live_cbr(S.pictures(S.run(L.LIVE_CBR, L.live_cbr())))


def test_cqp_set_qp_during_motion_and_paintover_burst():
    L.check_live_cqp(S.pictures(S.run(L.LIVE_CQP, L.live_cqp())))


@pytest.mark.parametrize("ring_slots", [2, 4, 16])
@pytest.mark.parametrize("rc_mode", [S.CQP, S.CBR], ids=["cqp", "cbr"])
def test_gop_and_idr_requests_in_flight(rc_mode, ring_slots):
    cfg = S.Config(L.W, L.H, rc_mode=rc_mode, kbps=500, fps=30.0, gop=10, ring_slots=ring_slots)
    L.check_gop(S.pictures(S.run(cfg, L.gop_script())))


@pytest.mark.parametrize("rc_mode", [S.CQP, S.CBR], ids=["cqp", "cbr"])
def test_resize_sequence_every_csc_path(rc_mode):
    """One session through 1:1, ragged, scaled (10 KB and 80 KB shared-memory tiles), the general scaled kernel, an upscale and
    back; every segment equals a fresh oracle encoder at the new size (in CBR a fresh rate controller) and starts with an IDR
    carrying an SPS of the new size."""
    segs = S.run(S.Config(L.W, L.H, rc_mode=rc_mode, kbps=300, fps=30.0), L.resize_script())
    assert [s.dst for s in segs] == [(dw, dh) for _, _, dw, dh in L.RESIZE_STEPS]
    assert [x.index for x in S.pictures(segs)] == list(range(len(L.RESIZE_STEPS) * L.RESIZE_PICTURES))


def _csc_80k(device):
    out = []
    for sw, sh, dw, dh in ((1920, 1080, 320, 180), (7680, 4320, 1280, 720)):
        f = synth.noise(sw, sh, 17)
        with Session(sw, sh, dst_width=dw, dst_height=dh, device=device, flags=N.B2V_FLAG_NO_ENCODE) as s:
            y, uv = s.csc_nv12(f)
        oy, ouv = oracle.csc_nv12(f, dst_w=dw, dst_h=dh)
        out.append(np.array_equal(y, oy) and np.array_equal(uv, ouv))
    return out


def test_scaled_80k_tier_on_a_second_device():
    """The 48-96 KB tier of the scaled CSC kernel needs an opt-in attribute, which CUDA applies per device: a session on a
    second GPU of the same process must get it too (device 0 first, then device 1)."""
    if N.lib().b2v_device_count() < 2:
        pytest.skip("one GPU visible")
    assert _csc_80k(0) == [True, True]
    assert _csc_80k(1) == [True, True]
    xs = S.pictures(S.run(S.Config(1920, 1080, 320, 180, rc_mode=S.CQP, qp=30),
                          [S.picture(L.desktop(1920, 1080, t)) for t in range(4)], device=1))
    assert len(xs) == 4
