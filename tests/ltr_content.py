"""Scripted desktop content for the long-term reference picture (B2V_FLAG_LONG_TERM_REF), on tests/synth.py's desktop: content that
goes away and comes back.  Every builder returns (frames, returns), `returns` being the indices of the pictures on which earlier
content comes back (the popup closes, the application switched away from is shown again)."""
import numpy as np

from tests import synth


def desktop(w, h, seed=1, invert=False):
    """A flat desktop as an office session shows it: a coloured background, a taskbar, two flat windows with title bars and a
    line of text-like glyphs.  Most macroblocks are flat, so a still picture is quiet: few co-located blocks fail the zero-motion
    exit."""
    rng = np.random.default_rng(seed)
    f = np.zeros((h, w, 4), np.uint8)
    f[..., :3] = (165, 110, 58) if not invert else (40, 90, 40)
    f[..., 3] = 255
    f[h - 32:, :, :3] = (40, 40, 40)
    for wx, wy, ww, wh in ((w // 16, h // 10, w // 2, h // 2), (w // 2, h // 3, w // 3, h // 2)):
        f[wy: wy + wh, wx: wx + ww, :3] = 236 if not invert else 30
        f[wy: wy + 22, wx: wx + ww, :3] = (150, 80, 40)
        for line in range(1):
            y = wy + 34 + 20 * line
            g = rng.integers(0, 2, (6, (ww - 40) // 2), dtype=np.uint8).repeat(2, 0).repeat(2, 1)
            f[y: y + 12, wx + 16: wx + 16 + g.shape[1], :3] = np.where(g > 0, 20, f[y, wx + 16, 0])[..., None]
    return f


def _typing(f, k, x0, y0):
    """k characters typed into f at (x0, y0): 8 x 12 px dark blocks, a few macroblocks per picture"""
    for i in range(k):
        x = x0 + 10 * i
        f[y0: y0 + 12, x: x + 8, :3] = (20 + 7 * i) % 90
    return f


def popup(w, h, before=3, open_for=4, after=3, seed=1):
    """A still desktop, a dialog box that opens over most of it, stays, and closes: `returns` = the closing picture."""
    base = desktop(w, h, seed)
    rng = np.random.default_rng(seed + 10)
    box = np.zeros((h * 3 // 16 * 4, w * 3 // 16 * 4, 4), np.uint8)
    box[..., :3] = rng.integers(0, 2, (box.shape[0] // 4, box.shape[1] // 4, 1), dtype=np.uint8).repeat(4, 0).repeat(4, 1) * 200 + 30
    box[:24, :, :3] = (120, 60, 20)
    box[..., 3] = 255
    frames = [base.copy() for _ in range(before)]
    for i in range(open_for):
        f = base.copy()
        f[h // 8: h // 8 + box.shape[0], w // 8: w // 8 + box.shape[1]] = box
        frames.append(_typing(f, i, w // 8 + 16, h // 8 + 40))
    frames += [base.copy() for _ in range(after)]
    return frames, [before + open_for]


def alt_tab(w, h, each=3, switches=3):
    """Two applications A and B shown in turn, A -> B -> A -> B, with typing (a few macroblocks per picture) in between:
    `returns` = every switch back to an application already seen."""
    apps = [desktop(w, h, 1), desktop(w, h, 4, invert=True)]
    frames, returns, typed = [], [], [0, 0]
    for s in range(switches + 1):
        a = s & 1
        if s >= 2:
            returns.append(len(frames))
        for _ in range(each):
            typed[a] += 1
            frames.append(_typing(apps[a].copy(), typed[a], w // 5, h // 3 + 16 * a))
    return frames, returns


def drag(w, h, n=10, step=24):
    """A window dragged across a textured desktop by `step` px per picture: the desktop behind it comes back."""
    rng = np.random.default_rng(3)
    base = desktop(w, h, 2)
    base[h - 32:, :, :3] = rng.integers(100, 200, (32, w, 1), dtype=np.uint8)
    win = np.zeros((h // 3, w // 3, 4), np.uint8)
    win[..., :3] = rng.integers(0, 2, (h // 3, w // 3, 1), dtype=np.uint8) * 180 + 40
    win[:20, :, :3] = (150, 80, 40)
    win[..., 3] = 255
    frames = []
    for t in range(n):
        f = base.copy()
        x = min(16 + step * t, w - win.shape[1])
        f[h // 3: h // 3 + win.shape[0], x: x + win.shape[1]] = win
        frames.append(f)
    return frames, []


def scroll(w, h, n=8):
    """synth.desktop's text region scrolling 8 px per picture."""
    return [synth.desktop(w, h, t) for t in range(n)], []


def caret(w, h, n=10):
    """A quiet desktop with a blinking caret: 2 x 16 px, on for two pictures, off for two."""
    base = desktop(w, h, 5)
    frames = []
    for t in range(n):
        f = base.copy()
        if (t // 2) & 1:
            f[h // 2: h // 2 + 16, w // 3: w // 3 + 2, :3] = 0
        frames.append(f)
    return frames, []


CONTENTS = {"popup": popup, "alt_tab": alt_tab, "drag": drag, "scroll": scroll, "caret": caret}
