"""The long-stream and live-control scripts (tests/longrun_scripts.py) run through the oracle alone: each reaches the regime it
is meant to pin on the GPU — frame_num wraps, paint-over bursts re-armed, the rate controller's clamps and debt rule, a QP
that moves after every control step, the GOP rule.  Parameters that miss their regime fail here, without a GPU."""
import pytest

from tests import longrun_scripts as L
from tests import scenario as S

CASES = [
    ("fullframe_cqp", L.FULLFRAME_CQP, L.fullframe_cqp, L.check_fullframe_cqp),
    ("striped", L.STRIPED, L.striped, L.check_striped),
    ("cbr_pinned", L.CBR_PINNED, L.cbr_pinned, L.check_cbr_pinned),
    ("cbr_generous", L.CBR_GENEROUS, L.cbr_generous, L.check_cbr_generous),
    ("cbr_debt", L.CBR_DEBT, L.cbr_debt, L.check_cbr_debt),
    ("live_cbr", L.LIVE_CBR, L.live_cbr, L.check_live_cbr),
    ("live_cqp", L.LIVE_CQP, L.live_cqp, L.check_live_cqp),
    ("gop_cqp", S.Config(L.W, L.H, rc_mode=S.CQP, gop=10), L.gop_script, L.check_gop),
    ("gop_cbr", S.Config(L.W, L.H, rc_mode=S.CBR, kbps=500, fps=30.0, gop=10), L.gop_script, L.check_gop),
]


@pytest.mark.parametrize("name,cfg,script,check", CASES, ids=[c[0] for c in CASES])
def test_script_reaches_its_regime(name, cfg, script, check):
    check(S.pictures(S.run(cfg, script(), gpu=False)))


def test_resize_script_restarts_every_segment():
    for rc_mode in (S.CQP, S.CBR):
        segs = S.run(S.Config(L.W, L.H, rc_mode=rc_mode, kbps=300, fps=30.0), L.resize_script(), gpu=False)
        assert [s.dst for s in segs] == [(dw, dh) for _, _, dw, dh in L.RESIZE_STEPS]
        for s in segs:
            assert [x.is_key for x in s.pictures] == [True] + [False] * (L.RESIZE_PICTURES - 1)
            assert [x.index for x in s.pictures] == list(range(s.first, s.first + L.RESIZE_PICTURES))      # frame ids continue


def test_driver_mirrors_the_host_idr_rule():
    """The oracle side's IDR decision and target_bits arithmetic (b2v_api.cu submit_common), on a script of controls alone."""
    ev = [S.set_gop(3)] + [S.picture(L.desktop(64, 48, t)) for t in range(7)] + [S.request_idr(), S.set_fps(24), S.set_bitrate(77)]
    ev += [S.picture(L.desktop(64, 48, 7)), S.set_gop(0), S.picture(L.desktop(64, 48, 8))]
    xs = S.pictures(S.run(S.Config(64, 48, rc_mode=S.CBR, kbps=100, fps=30.0), ev, gpu=False))
    assert [x.is_key for x in xs] == [True, False, False, True, False, False, True, True, False]
    assert [x.target_bits for x in xs] == [3333] * 7 + [3208] * 2
    assert xs[7].after.startswith("set_bitrate(77)")
