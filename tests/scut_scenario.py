"""Scene cuts through the two-sided driver of tests/scenario.py: the oracle side is tests/ltr_scenario.py's on a SceneCutEncoder
(oracle/scut.py), with scene cuts turned on at creation and after every resize when Config.flags carries B2V_FLAG_SCENE_CUT (after
droppable pictures, wide motion and the long-term reference, when those are on too).  Nothing else changes: the same events, the
same comparisons.  Combines with the device and tensor drivers."""
from __future__ import annotations

from contextlib import contextmanager
from unittest import mock

from oracle.scut import SceneCutEncoder
from tests import ltr_scenario as LS
from tests import scenario

FLAG_SCENE_CUT = 2048            # = selkies_b200._native.B2V_FLAG_SCENE_CUT (the oracle side needs no library)


class ScutOracleSide(LS.LtrOracleSide):
    def _new_encoder(self, sw, sh, dw, dh):
        with mock.patch.object(LS, "LongTermRefEncoder", SceneCutEncoder):
            super()._new_encoder(sw, sh, dw, dh)
        if self.cfg.flags & FLAG_SCENE_CUT:
            self.enc.set_scene_cut(True)


@contextmanager
def oracle_side():
    """scenario.run with ScutOracleSide as its oracle side for the duration of the block."""
    with mock.patch.object(scenario, "OracleSide", ScutOracleSide):
        yield


def run(cfg: scenario.Config, events, **kw) -> list:
    with oracle_side():
        return scenario.run(cfg, events, **kw)


def switches(w, h):
    """A stream of whole-screen changes and the pictures after them: the pairs of the scene-cut table (include/b2video.h,
    INTEGRATION.md), each switch followed by a still picture (which stays P)."""
    from tests import ltr_content as LC
    from tests import synth
    a, b = LC.desktop(w, h, 1), LC.desktop(w, h, 1, invert=True)
    return [a, a, b, b, synth.desktop(w, h), synth.bars(w, h), synth.bars(w, h), synth.gradient(w, h), synth.desktop(w, h),
            synth.desktop(w, h, seed=2), synth.noise(w, h, 0), synth.noise(w, h, 1), a]
