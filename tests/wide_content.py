"""Seeded fast-motion contents for wide-range motion (B2V_FLAG_WIDE_MOTION): tests/synth.py's desktop with its text region scrolled
at any speed, and a textured window dragged across the still desktop.  Each picture carries its true displacement."""
import numpy as np

from tests import synth


def desktop_scroll(w, h, t, speed, seed=1):
    """synth.desktop with the text region scrolled up by `speed` px per picture (speed 8 is synth.desktop itself).  Content at (x, y)
    was at (x, y + speed) one picture earlier: true vector (0, +speed) px for the region, rows from h - speed on are revealed."""
    rng = np.random.default_rng(seed)
    f = np.zeros((h, w, 4), np.uint8)
    f[..., :3] = (240, 240, 240)
    f[..., 3] = 255
    f[: h // 12, :, :3] = (60, 40, 30)
    f[:, : w // 6, :3] = (200, 210, 220)
    th = 4 * h
    glyph = rng.integers(0, 2, (th // 2, (w - w // 6) // 2), dtype=np.uint8).repeat(2, 0).repeat(2, 1)
    line = ((np.arange(th) // 8) % 3 != 2)[:, None]
    txt = np.where((glyph[:th, : w - w // 6] > 0) & line, 20, 240).astype(np.uint8)
    y0 = h // 12
    off = (speed * t) % (th - h)
    region = txt[off: off + (h - y0), :]
    f[y0:, w // 6: w // 6 + region.shape[1], :3] = region[..., None]
    return f


def scroll_region(w, h, speed):
    """(x0, y0, x1, y1) of the scrolled area whose content was on screen one picture earlier (the revealed rows excluded)."""
    return w // 6, h // 12, w, h - speed


def window(ww=320, wh=240, seed=7):
    """A window: a title bar over text-like content, BGRA."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 2, ((wh + 1) // 2, (ww + 1) // 2), dtype=np.uint8).repeat(2, 0).repeat(2, 1)[:wh, :ww]
    f = np.zeros((wh, ww, 4), np.uint8)
    f[..., :3] = np.where(g > 0, 30, 235)[..., None]
    f[:20, :, :3] = (150, 80, 40)
    f[..., 3] = 255
    return f


def drag(w, h, t, v, start=(0, 0), ww=320, wh=240):
    """The still desktop with `window` at start + t * v (px; clipped at the picture's edges).  Window content at (x, y) was at
    (x, y) - v one picture earlier: true vector -v px."""
    f = synth.desktop(w, h, 0)
    win = window(ww, wh)
    x, y = start[0] + t * v[0], start[1] + t * v[1]
    xa, ya, xb, yb = max(x, 0), max(y, 0), min(x + ww, w), min(y + wh, h)
    if xa < xb and ya < yb:
        f[ya:yb, xa:xb] = win[ya - y:yb - y, xa - x:xb - x]
    return f


def drag_window_at(t, v, start=(0, 0), ww=320, wh=240):
    """(x0, y0, x1, y1) of the window in picture t."""
    x, y = start[0] + t * v[0], start[1] + t * v[1]
    return x, y, x + ww, y + wh


def interior_mbs(rect, w, h, margin=1):
    """Macroblocks (mbx, mby) lying inside rect and the picture with `margin` macroblocks to spare on every side."""
    x0, y0, x1, y1 = rect
    out = []
    for mby in range((h + 15) // 16):
        for mbx in range((w + 15) // 16):
            X, Y = mbx * 16, mby * 16
            if X >= x0 + 16 * margin and Y >= y0 + 16 * margin and X + 16 <= min(x1, w) - 16 * margin and Y + 16 <= min(y1, h) - 16 * margin:
                out.append((mbx, mby))
    return out
