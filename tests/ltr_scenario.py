"""The long-term reference picture through the two-sided driver of tests/scenario.py: the oracle side is tests/wide_scenario.py's on a
LongTermRefEncoder (oracle/ltr.py), with the long-term reference turned on at creation and after every resize when Config.flags
carries B2V_FLAG_LONG_TERM_REF (after wide motion, when that is on too).  Nothing else changes: the same events, the same
comparisons."""
from __future__ import annotations

from contextlib import contextmanager
from unittest import mock

from oracle.ltr import LongTermRefEncoder
from tests import scenario
from tests import wide_scenario as WS

FLAG_LONG_TERM_REF = 512         # = selkies_b200._native.B2V_FLAG_LONG_TERM_REF (the oracle side needs no library)


class LtrOracleSide(WS.WideOracleSide):
    def _new_encoder(self, sw, sh, dw, dh):
        with mock.patch.object(WS, "WideRefEncoder", LongTermRefEncoder):
            super()._new_encoder(sw, sh, dw, dh)
        if self.cfg.flags & FLAG_LONG_TERM_REF:
            self.enc.set_long_term_ref(True)


@contextmanager
def oracle_side():
    """scenario.run with LtrOracleSide as its oracle side for the duration of the block."""
    with mock.patch.object(scenario, "OracleSide", LtrOracleSide):
        yield


def run(cfg: scenario.Config, events, **kw) -> list:
    with oracle_side():
        return scenario.run(cfg, events, **kw)
