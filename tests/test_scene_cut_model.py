"""Scene cuts against the independent decisions model (tests/h264_model_scene_cut.py on tests/h264_model.py): on every P picture of
the oracle's streams, the model's two costs — from the source, libavcodec's decoding of the stream (the references) and the
independent reader's records of the previous picture (tests/h264_syntax_refs.py) — equal the oracle's, and the model names exactly
the pictures the oracle cut.  Contents: the switches of tests/scut_scenario.py, the scripts of tests/ltr_content.py and
tests/wide_content.py, with wide motion and the long-term reference on and off, at QP 26 and 36."""
import numpy as np
import pytest

import oracle
from oracle import avdec
from oracle.scut import SceneCutEncoder
from tests import h264_model as M
from tests import h264_model_scene_cut as MS
from tests import h264_syntax_refs as HSR
from tests import ltr_content as LC
from tests import scut_scenario as SC
from tests import wide_content as WC

W, H = 320, 192         # multiples of 16: the decoded pictures are the coded ones


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


def _contents():
    out = {k: LC.CONTENTS[k](W, H)[0] for k in ("popup", "alt_tab", "drag", "scroll")}
    out["switches"] = SC.switches(W, H)
    out["wide_scroll"] = [WC.desktop_scroll(W, H, t, 24) for t in range(5)]
    out["wide_drag"] = [WC.drag(W, H, t, (40, 16), (0, 0), 96, 64) for t in range(5)]
    return out


@pytest.mark.parametrize("wide", [False, True], ids=["", "wide"])
@pytest.mark.parametrize("ltr", [False, True], ids=["", "ltr"])
@pytest.mark.parametrize("qp", [26, 36])
def test_model_names_the_oracles_cuts(qp, ltr, wide):
    named = 0
    for name, frames in _contents().items():
        e = SceneCutEncoder(W, H)
        e.set_wide_motion(wide)
        e.set_long_term_ref(ltr)
        e.set_scene_cut(True)
        aus, states, srcs = [], [], []
        for i, f in enumerate(frames):
            aus.append(e.encode_bgra(f, i == 0, rc_mode=1, qp=qp))
            states.append(e.scut_state())
            srcs.append(oracle.csc_nv12(f)[0])
        e.close()
        pics = HSR.parse_stream(aus)
        recs = [np.asarray(y) for y, _, _ in avdec.decode_stream(aus, quiet=True)]
        for k in range(1, len(frames)):
            lt = pics[k - 1].long_term[0] if pics[k - 1].long_term else None
            dec = (M.decimate(srcs[k]), M.decimate(srcs[k - 1])) if wide else None
            intra, inter = MS.picture_costs(srcs[k], recs[k - 1], None if lt is None else recs[lt], pics[k - 1].mbs, qp, wide, dec)
            where = f"{name} picture {k}"
            assert (intra, inter) == (states[k]["cost_intra"], states[k]["cost_inter"]), (where, intra, inter, states[k])
            assert MS.cuts(intra, inter) == bool(states[k]["cut"]), where
            named += MS.cuts(intra, inter)
    assert named > 0
