"""Wide-range motion through the two-sided driver of tests/scenario.py: the oracle side is tests/layered_scenario.py's (droppable when
the session is) on a WideRefEncoder (oracle/wide.py), with wide motion turned on at creation and after every resize when Config.flags
carries B2V_FLAG_WIDE_MOTION.
Nothing else changes: the same events, the same comparisons.  Combines with the device and tensor drivers."""
from __future__ import annotations

from contextlib import contextmanager
from unittest import mock

from oracle.wide import WideRefEncoder
from tests import layered_scenario as LS
from tests import scenario

FLAG_WIDE_MOTION = 256           # = selkies_b200._native.B2V_FLAG_WIDE_MOTION (the oracle side needs no library)


class WideOracleSide(LS.LayeredOracleSide):
    def _new_encoder(self, sw, sh, dw, dh):
        with mock.patch.object(LS, "LayeredRefEncoder", WideRefEncoder):
            super()._new_encoder(sw, sh, dw, dh)
        if self.cfg.flags & FLAG_WIDE_MOTION:
            self.enc.set_wide_motion(True)


@contextmanager
def oracle_side():
    """scenario.run with WideOracleSide as its oracle side for the duration of the block."""
    with mock.patch.object(scenario, "OracleSide", WideOracleSide):
        yield


def run(cfg: scenario.Config, events, **kw) -> list:
    with oracle_side():
        return scenario.run(cfg, events, **kw)
