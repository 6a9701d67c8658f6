"""Damage-rectangle ingest (B2V_FLAG_DAMAGE) through the two-sided driver of tests/scenario.py.  The oracle side does not change:
it is fed whole frames.  The GPU side's session has the flag; each picture's rectangles are computed from the frame before it
(`damage`), and before every ring submit the slot is filled with random bytes and then only the rectangles are written, so a
single byte read from outside them would change the access units.  The first picture, and the first after a resize, is
submitted whole.  Also the desktop contents the tests feed: typing, a scrolling pane, a window drag, a cut, an unchanged
picture and a full change."""
from __future__ import annotations

import dataclasses
from contextlib import contextmanager
from unittest import mock

import numpy as np

from tests import scenario, synth

DAMAGE = 1024          # = selkies_b200._native.B2V_FLAG_DAMAGE
CELL = 8               # damage is found on an 8 x 8 grid: rectangles that do not line up with the 16 x 16 tiles


def damage(prev: np.ndarray, cur: np.ndarray) -> list:
    """(x, y, w, h) rectangles covering every pixel of `cur` that differs from `prev`: runs of changed 8 x 8 cells per cell row
    (clipped to the frame); an empty list when nothing changed."""
    h, w = cur.shape[:2]
    diff = (prev != cur).any(axis=2)
    ch, cw = -(-h // CELL), -(-w // CELL)
    pad = np.zeros((ch * CELL, cw * CELL), bool)
    pad[:h, :w] = diff
    cells = pad.reshape(ch, CELL, cw, CELL).any(axis=(1, 3))
    out = []
    for cy in range(ch):
        row = np.concatenate(([False], cells[cy], [False]))
        edges = np.flatnonzero(row[1:] != row[:-1])
        for a, b in zip(edges[::2], edges[1::2]):
            x0, y0 = a * CELL, cy * CELL
            out.append((int(x0), int(y0), int(min(b * CELL, w) - x0), int(min(y0 + CELL, h) - y0)))
    return out


def submit_poisoned(s, frame: np.ndarray, rects, rng) -> None:
    """Ring submit of `frame` with `rects` (None: whole) into a slot that holds random bytes outside them.  More rectangles than
    the library takes are merged first (Session.normalize_rects): what is written is what is submitted."""
    from selkies_b200 import _native as N
    from selkies_b200.session import normalize_rects
    slot, view = s.acquire()
    view[...] = rng.integers(0, 256, view.shape, dtype=np.uint8)
    if rects is not None:
        rects = normalize_rects(rects, frame.shape[1], frame.shape[0])
        for x, y, w, h in rects:
            view[y:y + h, x:x + w] = frame[y:y + h, x:x + w]
        try:
            s.submit_slot(slot, damage=rects)
            return
        except N.B2VError as e:
            if e.code != N.B2V_ESTATE:
                raise
    view[...] = frame
    s.submit_slot(slot)


class DamageGpuSide(scenario.GpuSide):
    def __init__(self, cfg: scenario.Config, device: int = 0):
        super().__init__(dataclasses.replace(cfg, flags=cfg.flags | DAMAGE, entry="ring"), device)
        self.prev, self.rng = None, np.random.default_rng(1)

    def control(self, ev):
        super().control(ev)
        if ev[0] == "resize":
            self.prev = None

    def picture(self, frame):
        rects = None if self.prev is None else damage(self.prev, frame)
        self.prev = frame
        submit_poisoned(self.s, frame, rects, self.rng)


@contextmanager
def gpu_side(cls=DamageGpuSide):
    with mock.patch.object(scenario, "GpuSide", cls):
        yield


def run(cfg: scenario.Config, events, **kw) -> list:
    """scenario.run with damage submits on the GPU side."""
    with gpu_side():
        return scenario.run(cfg, events, **kw)


# ---- contents ------------------------------------------------------------------------------------------------------------------
def desktop_session(w: int, h: int, seed: int = 0) -> list:
    """A desktop through typing, a scrolling pane of about a third of the screen, a window drag, an unchanged picture, a cut, a
    full change and a picture after it: one frame each (the unchanged picture is the same object as the one before)."""
    rng = np.random.default_rng(seed)
    frames = [synth.desktop(w, h, 0)]

    def step(fn):
        g = frames[-1].copy()
        fn(g)
        frames.append(g)

    def typing(g):                       # a few glyph-sized cells along a text line
        y = int(rng.integers(h // 8, max(h // 8 + 1, h - 12)))
        for k in range(int(rng.integers(1, 5))):
            x = int(rng.integers(0, max(1, w - 7)))
            g[y:y + 11, x:x + 7, :3] = rng.integers(0, 256, (min(11, h - y), min(7, w - x), 3), dtype=np.uint8)

    pane = (w // 3, h // 4, min(w - w // 3, max(16, w // 2)), min(h - h // 4, max(16, h * 2 // 3)))   # x, y, width, height: about a third of the screen

    def scroll(g):
        x, y, pw, ph = pane
        g[y:y + ph - 8, x:x + pw] = g[y + 8:y + ph, x:x + pw]
        g[y + ph - 8:y + ph, x:x + pw, :3] = rng.integers(0, 256, (8, pw, 3), dtype=np.uint8)

    win = synth.noise(max(8, w // 5), max(8, h // 5), 9)
    ww, wh = win.shape[1], win.shape[0]

    def drag(k):
        def f(g):
            g[...] = frames[0]
            x, y = min(w - ww, 5 + 13 * k), min(h - wh, 3 + 7 * k)
            g[y:y + wh, x:x + ww] = win
        return f

    for _ in range(3):
        step(typing)
    step(scroll)
    step(scroll)
    for k in range(3):
        step(drag(k))
    frames.append(frames[-1])            # unchanged: an empty list
    frames.append(synth.desktop(w, h, 3, seed=4))       # a cut
    frames.append(synth.noise(w, h, 2))                 # a full change
    step(typing)
    return frames
