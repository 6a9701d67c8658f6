"""Droppable pictures through the two-sided driver of tests/scenario.py: the oracle side is a LayeredRefEncoder (oracle/layers.py),
set droppable at creation and after every resize when Config.flags carries B2V_FLAG_DROPPABLE.  Nothing else changes: the same
events, the same comparisons.  Combines with the device and tensor drivers, which replace the GPU side."""
from __future__ import annotations

from contextlib import contextmanager
from unittest import mock

import oracle
from oracle.layers import LayeredRefEncoder
from tests import scenario

FLAG_DROPPABLE = 128             # = selkies_b200._native.B2V_FLAG_DROPPABLE (the oracle side needs no library)


class LayeredOracleSide(scenario.OracleSide):
    def _new_encoder(self, sw, sh, dw, dh):
        with mock.patch.object(oracle, "RefEncoder", LayeredRefEncoder):
            super()._new_encoder(sw, sh, dw, dh)
        if self.cfg.flags & FLAG_DROPPABLE:
            self.enc.set_droppable(True)


@contextmanager
def oracle_side():
    """scenario.run with LayeredOracleSide as its oracle side for the duration of the block."""
    with mock.patch.object(scenario, "OracleSide", LayeredOracleSide):
        yield


def run(cfg: scenario.Config, events, **kw) -> list:
    with oracle_side():
        return scenario.run(cfg, events, **kw)
