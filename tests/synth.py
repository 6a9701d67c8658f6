"""Seeded synthetic BGRA inputs (SURVEY.md §8d: S1 bars+box, S2 random, S3 desktop-like, S4 gradient pan)."""
import numpy as np

BARS_RGB = [(255, 255, 255), (255, 255, 0), (0, 255, 255), (0, 255, 0), (255, 0, 255), (255, 0, 0), (0, 0, 255), (0, 0, 0)]


def bars(w, h, t=0):
    f = np.zeros((h, w, 4), np.uint8)
    f[..., 3] = 255
    bw = max(1, w // 8)
    for i, (r, g, b) in enumerate(BARS_RGB):
        f[:, i * bw:(i + 1) * bw if i < 7 else w, :3] = (b, g, r)
    bs = min(64, h // 2, w // 2)
    x = (t * 4) % max(1, w - bs)
    y = (t * 3) % max(1, h - bs)
    f[y:y + bs, x:x + bs, :3] = (40, 200, 120)
    return f


def noise(w, h, seed=0):
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    f[..., 3] = 255
    return f


def gradient(w, h, t=0):
    x = (np.arange(w)[None, :] + 2 * t)
    y = np.arange(h)[:, None]
    f = np.zeros((h, w, 4), np.uint8)
    f[..., 0] = (x * 255 // max(1, w - 1)) % 256
    f[..., 1] = (y * 255 // max(1, h - 1)) % 256
    f[..., 2] = ((x + y) // 2) % 256
    f[..., 3] = 255
    return f


def desktop(w, h, t=0, seed=1):
    """Flat regions + 1-px text-like patterns + a region scrolling 8 px/frame."""
    rng = np.random.default_rng(seed)
    f = np.zeros((h, w, 4), np.uint8)
    f[..., :3] = (240, 240, 240)
    f[..., 3] = 255
    f[: h // 12, :, :3] = (60, 40, 30)                      # title bar
    f[:, : w // 6, :3] = (200, 210, 220)                    # side panel
    # text-like content, generated once as a tall strip and scrolled
    th = 4 * h
    glyph = rng.integers(0, 2, (th // 2, (w - w // 6) // 2), dtype=np.uint8).repeat(2, 0).repeat(2, 1)
    line = ((np.arange(th) // 8) % 3 != 2)[:, None]
    txt = np.where((glyph[:th, : w - w // 6] > 0) & line, 20, 240).astype(np.uint8)
    y0 = h // 12
    off = (8 * t) % (th - h)
    region = txt[off: off + (h - y0), :]
    f[y0:, w // 6: w // 6 + region.shape[1], 0] = region
    f[y0:, w // 6: w // 6 + region.shape[1], 1] = region
    f[y0:, w // 6: w // 6 + region.shape[1], 2] = region
    return f


def tiles(w, h, noise_at=(), light_at=(), seed=0, grey=130, base=None):
    """A flat grey field (or a copy of `base`) with 16x16 tiles at macroblock addresses (raster order, ceil(w / 16) macroblocks per
    row).  Grey 130 converts to Y = Cb = Cr = 128, which intra DC prediction reproduces exactly at any QP.  At the addresses of
    `noise_at`: uniform noise, I_PCM at QP 0 and 4 in IDR slices and in P pictures whose reference holds something else there; at
    those of `light_at`: a flat tile a few levels off grey, which costs a few bits.  Fresh noise per seed, so that a motion
    search never finds a tile of an earlier picture."""
    f = np.array(base) if base is not None else np.full((h, w, 4), grey, np.uint8)
    f[..., 3] = 255
    mbw = (w + 15) // 16
    rng = np.random.default_rng(seed)
    for a in noise_at:
        y, x = a // mbw * 16, a % mbw * 16
        f[y:y + 16, x:x + 16, :3] = rng.integers(0, 256, (16, 16, 3), dtype=np.uint8)[: h - y, : w - x]
    for k, a in enumerate(light_at):
        y, x = a // mbw * 16, a % mbw * 16
        f[y:y + 16, x:x + 16, :3] = grey + 6 + 2 * (seed % 5) + k % 3
    return f


def predictor_paths(w, h):
    """Eleven pictures that walk every exit of the P-picture motion search (DESIGN.md §5.3): a still (zero-motion exit), the same with
    +-2 LSB noise (zero-vector candidate), the onset of a scroll (anchors search, their groups take the anchor's vector), the scroll
    going on (temporal predictor), a cut to noise (new content: anchors search, the rest run the reduced search), noise again, and back
    to the still."""
    still = desktop(w, h, 0)

    def jitter(seed):
        rng = np.random.default_rng(seed)
        f = still.astype(np.int16)
        f[..., :3] += rng.integers(-2, 3, (h, w, 3), dtype=np.int16)
        return np.clip(f, 0, 255).astype(np.uint8)
    return ([still, still, jitter(1), jitter(2)] + [desktop(w, h, t) for t in (1, 2, 3)]
            + [noise(w, h, 40), noise(w, h, 41), still, still])
