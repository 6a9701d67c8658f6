"""The quality measurement of B2V_FLAG_QUALITY (include/b2video.h, b2v_quality) restated in numpy, and two independent float64
forms of its SSIM that the CPU tests hold it against.

`measure` is the statement the GPU must equal: exact int64 SSEs, and per 8x8 window on the 4-sample grid the integer window sums
and the fp64 expression evaluated in the stated order.  The 64-sample window sums come from 4x4 block sums here too, but in
int64, so they are the exact sums whatever way they are formed."""
from __future__ import annotations

import numpy as np

C1, C2 = 416, 235963            # round(0.01^2 255^2 64), round(0.03^2 255^2 64 63)


def ssim_windows(s: np.ndarray, r: np.ndarray) -> np.ndarray:
    """Per-window SSIM of two luma records (2-D uint8, same shape), windows with origins on the 4-sample grid that lie wholly
    inside; returns a (rows, cols) float64 array (empty when the record is below 8 samples either way)."""
    h, w = s.shape
    nby, nbx = h // 4, w // 4
    if nby < 2 or nbx < 2:
        return np.zeros((0, 0))
    s = s[: nby * 4, : nbx * 4].astype(np.int64)
    r = r[: nby * 4, : nbx * 4].astype(np.int64)

    def blocks(a):
        return a.reshape(nby, 4, nbx, 4).sum(axis=(1, 3))

    def windows(b):
        return b[:-1, :-1] + b[1:, :-1] + b[:-1, 1:] + b[1:, 1:]

    sx, sy = windows(blocks(s)), windows(blocks(r))
    q, p = windows(blocks(s * s + r * r)), windows(blocks(s * r))
    v = 64 * q - sx * sx - sy * sy
    c = 64 * p - sx * sy
    num = (2 * sx * sy + C1).astype(np.float64) * (2 * c + C2).astype(np.float64)
    den = (sx * sx + sy * sy + C1).astype(np.float64) * (v + C2).astype(np.float64)
    return num / den


def measure(s_y, s_uv, r_y, r_uv, dst_w: int, y_start: int, height: int) -> dict:
    """The measurement of the record at rows y_start .. y_start + height - 1, columns 0 .. dst_w - 1 of S (s_y, s_uv: NV12 planes,
    chroma interleaved) against R (r_y, r_uv).  The fields of b2v_quality."""
    ys, yr = s_y[y_start:y_start + height, :dst_w], r_y[y_start:y_start + height, :dst_w]
    cs = s_uv[y_start // 2:(y_start + height) // 2, :dst_w].astype(np.int64)
    cr = r_uv[y_start // 2:(y_start + height) // 2, :dst_w].astype(np.int64)
    d = ys.astype(np.int64) - yr.astype(np.int64)
    dc = cs - cr
    win = ssim_windows(ys, yr)
    n = int(win.size)
    return {"sse_y": int((d * d).sum()), "sse_cb": int((dc[:, 0::2] ** 2).sum()), "sse_cr": int((dc[:, 1::2] ** 2).sum()),
            "samples_y": dst_w * height, "samples_c": dst_w * height // 4,
            "ssim_y": float(win.mean()) if n else float("nan"), "ssim_windows": n}


def ssim_direct(s: np.ndarray, r: np.ndarray) -> np.ndarray:
    """Per-window SSIM by loops over the windows, from each window's 64 samples: means, unbiased variances and covariance in
    float64, in the textbook form with the constants of the statement (C1 / 64^2 on the means, C2 / (64 * 63) on the
    variances)."""
    h, w = s.shape
    rows, cols = max(0, (h - 8) // 4 + 1), max(0, (w - 8) // 4 + 1)
    out = np.zeros((rows, cols))
    c1, c2 = C1 / 4096.0, C2 / 4032.0
    for j in range(rows):
        for i in range(cols):
            a = s[4 * j:4 * j + 8, 4 * i:4 * i + 8].astype(np.float64).ravel()
            b = r[4 * j:4 * j + 8, 4 * i:4 * i + 8].astype(np.float64).ravel()
            ma, mb = a.mean(), b.mean()
            va, vb = a.var(ddof=1), b.var(ddof=1)
            cab = ((a - ma) * (b - mb)).sum() / 63.0
            out[j, i] = ((2 * ma * mb + c1) * (2 * cab + c2)) / ((ma * ma + mb * mb + c1) * (va + vb + c2))
    return out


def ssim_boxfilter(s: np.ndarray, r: np.ndarray) -> np.ndarray:
    """Per-window SSIM from 8x8 box sums of float64 images (scipy.ndimage), sampled on the 4-sample grid."""
    from scipy import ndimage

    h, w = s.shape
    rows, cols = max(0, (h - 8) // 4 + 1), max(0, (w - 8) // 4 + 1)
    if not rows or not cols:
        return np.zeros((0, 0))
    a, b = s.astype(np.float64), r.astype(np.float64)
    k = np.ones((8, 8))

    def box(x):
        # origin (-4, -4): output (y, x) is the sum over rows y .. y + 7 and columns x .. x + 7
        full = ndimage.correlate(x, k, mode="constant", origin=(-4, -4))
        return full[0:4 * rows:4, 0:4 * cols:4]

    sx, sy, sxx, syy, sxy = box(a), box(b), box(a * a), box(b * b), box(a * b)
    mx, my = sx / 64, sy / 64
    vx, vy = (sxx - sx * sx / 64) / 63, (syy - sy * sy / 64) / 63
    cxy = (sxy - sx * sy / 64) / 63
    c1, c2 = C1 / 4096.0, C2 / 4032.0
    return ((2 * mx * my + c1) * (2 * cxy + c2)) / ((mx * mx + my * my + c1) * (vx + vy + c2))
