"""GPU parity over long streams (tests/scenario.py driver, scripts in tests/longrun_scripts.py): hundreds of pictures submitted
without a flush, every access unit, QP, key flag and frame id equal to the oracle's, the reconstruction equal at the end and
the stream decoded by libavcodec to it.  What only shows over time: frame_num wrapping at 256 (in striped mode per band, advanced
only when the band is delivered), paint-over re-arming across many still/motion cycles, and the rate controller's clamps
(fullness in [-4T, 64T], QP in [10, 51]) and its debt rule."""
import pytest

from tests import longrun_scripts as L
from tests import scenario as S

pytestmark = pytest.mark.gpu


def test_fullframe_cqp_600_pictures_paintover_frame_num_wraps():
    xs = S.pictures(S.run(L.FULLFRAME_CQP, L.fullframe_cqp()))
    L.check_fullframe_cqp(xs)


def test_striped_4_bands_300_pictures_band_frame_num():
    xs = S.pictures(S.run(L.STRIPED, L.striped()))
    L.check_striped(xs)


@pytest.mark.parametrize("cfg,script,check", [(L.CBR_PINNED, L.cbr_pinned, L.check_cbr_pinned),
                                              (L.CBR_GENEROUS, L.cbr_generous, L.check_cbr_generous),
                                              (L.CBR_DEBT, L.cbr_debt, L.check_cbr_debt)], ids=["qp51_full64T", "qp10_fullm4T", "debt_rule"])
def test_cbr_regime(cfg, script, check):
    check(S.pictures(S.run(cfg, script())))


def test_1080p_cbr_desktop_scroll_120_pictures():
    xs = S.pictures(S.run(L.HD, L.hd_scroll()))
    assert len(xs) == L.HD_PICTURES and len({x.qp for x in xs}) > 3
