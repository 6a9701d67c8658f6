"""Device-frame ingest through the two-sided driver of tests/scenario.py.  Nothing about the oracle side changes: it is fed the
BGRA frame.  On the GPU side each distinct frame object is uploaded once, as the resident entry does, but into a torch tensor
holding the frame's channels in the order of `DeviceConfig.pixel_format`.  With a `margin` the frame sits that many pixels inside
a larger surface.  Every picture is submitted with b2v_submit_device (Session.submit_device) on torch's current stream."""
from __future__ import annotations

import dataclasses
from contextlib import contextmanager
from dataclasses import dataclass
from unittest import mock

import numpy as np

from tests import scenario

# BGRA frame -> channels of each pixel format, in memory order
CHANNELS = {"BGRA": [0, 1, 2, 3], "RGBA": [2, 1, 0, 3], "BGR": [0, 1, 2], "RGB": [2, 1, 0]}


def reorder(bgra, pixel_format: str) -> np.ndarray:
    """The (H, W, 4) BGRA frame as (H, W, 4 or 3) pixels of `pixel_format`."""
    return np.ascontiguousarray(bgra[..., CHANNELS[pixel_format]])


def device_surface(bgra, pixel_format: str = "BGRA", margin=(0, 0), device: int = 0, fill: int = 0x5A):
    """A torch uint8 tensor on cuda:`device` holding `bgra` reordered to `pixel_format` at (x, y) = margin, inside a surface
    with as many pixels of `fill` after the frame as before it."""
    import torch
    h, w = bgra.shape[:2]
    mx, my = margin
    px = reorder(bgra, pixel_format)
    t = torch.full((h + 2 * my, w + 2 * mx, px.shape[2]), fill, dtype=torch.uint8, device=f"cuda:{device}")
    t[my:my + h, mx:mx + w] = torch.from_numpy(px).to(t.device)
    return t


@dataclass
class DeviceConfig(scenario.Config):
    pixel_format: str = "BGRA"         # byte order of the tensor (BGRA, RGBA, BGR, RGB)
    margin: tuple = (0, 0)             # (left, top) pixels of surface before the frame; as many after it, so the row stride is
                                       # (width + 2 * left) pixels


class DeviceGpuSide(scenario.GpuSide):
    def __init__(self, cfg: DeviceConfig, device: int = 0):
        super().__init__(dataclasses.replace(cfg, entry="ring"), device)     # the session; pictures take the device path below
        self.cfg, self.device = cfg, device

    def picture(self, frame):
        if id(frame) not in self.uploaded:       # held with the frame, so that its id stays unique; a resize clears it
            self.uploaded[id(frame)] = (device_surface(frame, self.cfg.pixel_format, self.cfg.margin, self.device), frame)
        self.s.submit_device(self.uploaded[id(frame)][0], pixel_format=self.cfg.pixel_format, origin=self.cfg.margin)


@contextmanager
def gpu_side(cls=DeviceGpuSide):
    """scenario.run with `cls` as its GPU side for the duration of the block."""
    with mock.patch.object(scenario, "GpuSide", cls):
        yield


def run(cfg: DeviceConfig, events, **kw) -> list:
    """scenario.run with device-frame submits on the GPU side."""
    with gpu_side():
        return scenario.run(cfg, events, **kw)
