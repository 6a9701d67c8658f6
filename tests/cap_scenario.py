"""The picture size cap through the two-sided driver of tests/scenario.py: the oracle side is tests/scut_scenario.py's on a
SizeCapEncoder (oracle/cap.py), with the cap turned on at creation and after every resize when Config.flags carries
B2V_FLAG_SIZE_CAP (scene cuts then go with it); one more event, set_max_picture_bytes(n), sets the cap on both sides from the next
picture on.  Combines with the device and tensor drivers."""
from __future__ import annotations

import dataclasses
from contextlib import contextmanager
from unittest import mock

from oracle.cap import SizeCapEncoder
from tests import scenario
from tests import scut_scenario as SC

FLAG_SIZE_CAP = 4096             # = selkies_b200._native.B2V_FLAG_SIZE_CAP (the oracle side needs no library)


def set_max_picture_bytes(n):
    return ("set_max_picture_bytes", n)


class CapOracleSide(SC.ScutOracleSide):
    def _new_encoder(self, sw, sh, dw, dh):
        cap = self.cfg.flags & FLAG_SIZE_CAP
        flags = self.cfg.flags
        if cap:      # scene cuts are an argument of set_size_cap
            self.cfg = dataclasses.replace(self.cfg, flags=flags & ~SC.FLAG_SCENE_CUT)
        with mock.patch.object(SC, "SceneCutEncoder", SizeCapEncoder):
            super()._new_encoder(sw, sh, dw, dh)
        self.cfg = dataclasses.replace(self.cfg, flags=flags)
        if cap:
            self.enc.set_size_cap(True, bool(flags & SC.FLAG_SCENE_CUT))
            self.enc.max_picture_bytes = getattr(self, "max_picture_bytes", 0)

    def control(self, ev):
        if ev[0] == "set_max_picture_bytes":
            self.max_picture_bytes = ev[1]
            self.enc.max_picture_bytes = ev[1]
        else:
            super().control(ev)


_gpu_control = scenario.GpuSide.control


def _cap_gpu_control(self, ev):
    if ev[0] == "set_max_picture_bytes":
        self.s.set_max_picture_bytes(ev[1])
    else:
        _gpu_control(self, ev)


@contextmanager
def oracle_side():
    """scenario.run with CapOracleSide, and a GPU side (any driver's) that takes set_max_picture_bytes, for the duration of the block."""
    with mock.patch.object(scenario, "OracleSide", CapOracleSide), mock.patch.object(scenario.GpuSide, "control", _cap_gpu_control):
        yield


def run(cfg: scenario.Config, events, **kw) -> list:
    with oracle_side():
        return scenario.run(cfg, events, **kw)
