"""Event scripts of the long-stream and live-control parity tests (tests/scenario.py events).  Shared by the GPU tests and by
tests/test_longrun_oracle.py, which runs them through the oracle alone and checks that every regime they are meant to reach
is reached — parameters that miss their regime fail without a GPU."""
from functools import lru_cache

import numpy as np

from tests import synth
from tests.scenario import (CBR, CQP, Config, picture, request_idr, resize, set_bitrate, set_fps, set_gop, set_qp)

W, H = 320, 192          # the desktop scroll restarts every 72 pictures at this height


@lru_cache(maxsize=96)
def desktop(w, h, t):
    f = synth.desktop(w, h, t)
    f.flags.writeable = False
    return f


@lru_cache(maxsize=96)
def noise(w, h, seed):
    f = synth.noise(w, h, seed)
    f.flags.writeable = False
    return f


# ---- long streams -------------------------------------------------------------------------------------------------------
FULLFRAME_CQP = Config(W, H, rc_mode=CQP, qp=30, paint=(3, 20, 2))


def fullframe_cqp():
    """About 600 pictures, one IDR: a scroll (restarting every 72 pictures), a still long enough for a paint-over burst, a cut
    to noise, a still of the noise (another burst), ten times over.  frame_num wraps twice."""
    t = 0
    for cycle in range(10):
        for _ in range(40):
            yield picture(desktop(W, H, t))
            t += 1
        for _ in range(9):
            yield picture(desktop(W, H, t - 1))
        yield picture(noise(W, H, cycle))
        for _ in range(10):
            yield picture(noise(W, H, cycle))


STRIPED = Config(W, H, rc_mode=CQP, qp=28, stripe_rows=3)
STRIPED_PICTURES = 300


def striped():
    """4 bands of 48 rows: band 0 changes every picture, band 1 every 7th, band 2 never after the IDR, band 3 every 2nd.
    Only band 0 wraps its frame_num."""
    for t in range(STRIPED_PICTURES):
        f = np.array(desktop(W, H, 0))
        f[0:48] = desktop(W, H, t)[0:48]
        f[48:96] = desktop(W, H, t // 7)[48:96]
        f[144:192] = desktop(W, H, t // 2)[144:192]
        yield picture(f)


# CBR regimes (30 pictures/s): the controller's clamps and the debt rule
CBR_PINNED = Config(W, H, rc_mode=CBR, kbps=40, fps=30.0)


def cbr_pinned():
    """Noise at 40 kbit/s: QP pinned at 51, fullness clamped at 64 pictures' budget; then a still desktop drains the bucket
    (how fast depends on the clamp) and a slow scroll follows."""
    for i in range(90):
        yield picture(noise(W, H, 100 + i))
    for _ in range(100):
        yield picture(desktop(W, H, 0))
    for t in range(40):
        yield picture(desktop(W, H, t // 4))


CBR_GENEROUS = Config(W, H, rc_mode=CBR, kbps=20000, fps=30.0)


def cbr_generous():
    """A still desktop with a small change every 5th picture at 20 Mbit/s: QP down to 10, fullness clamped at -4 pictures."""
    base = desktop(W, H, 0)
    for i in range(150):
        f = base
        if i % 5 == 4:
            f = np.array(base)
            f[100:116, 100:164, :3] = (i * 37) % 256
        yield picture(f)


CBR_DEBT = Config(W, H, rc_mode=CBR, kbps=600, fps=30.0)


def cbr_debt():
    """A scroll that jumps to a new position every 6 pictures: every jump is a spike the two-picture rule lets through, and
    at 600 kbit/s they pile up more than RC_DEBT_PICTURES pictures' worth of debt."""
    for i in range(200):
        yield picture(desktop(W, H, (i // 6) * 37 + i % 6))


HD = Config(1920, 1080, rc_mode=CBR, kbps=6000, fps=60.0)
HD_PICTURES = 120


def hd_scroll():
    for t in range(HD_PICTURES):
        yield picture(synth.desktop(1920, 1080, t))


# ---- live control -------------------------------------------------------------------------------------------------------
LIVE_CBR = Config(W, H, rc_mode=CBR, kbps=150, fps=30.0)
LIVE_CBR_STEPS = {"up": 25, "down": 45, "idr": 65, "remb": 80, "fps60": 100, "fps24": 110}


def live_cbr():
    """About 120 pictures of scroll with bitrate steps: x10 up, /20 down, a change on the picture of a requested IDR, a change on
    every picture for 10 pictures (REMB burst), then the frame rate 30 -> 60 -> 24."""
    s = LIVE_CBR_STEPS
    for t in range(125):
        if t == s["up"]:
            yield set_bitrate(1500)
        if t == s["down"]:
            yield set_bitrate(75)
        if t == s["idr"]:
            yield set_bitrate(200)
            yield request_idr()
        if s["remb"] <= t < s["remb"] + 10:
            yield set_bitrate(260 - 6 * (t - s["remb"]))
        if t == s["fps60"]:
            yield set_fps(60)
        if t == s["fps24"]:
            yield set_fps(24)
        yield picture(desktop(W, H, t))


LIVE_CQP = Config(W, H, rc_mode=CQP, qp=30, paint=(3, 20, 4))


def live_cqp():
    """set_qp during motion (pictures 6, 12) and in the middle of a scheduled paint-over burst."""
    for t in range(20):
        if t == 6:
            yield set_qp(24)
        if t == 12:
            yield set_qp(36)
        yield picture(desktop(W, H, t))
    for i in range(14):
        if i == 5:
            yield set_qp(33)
        yield picture(desktop(W, H, 19))
    for t in range(20, 26):
        yield picture(desktop(W, H, t))


GOP_KEYS = [0, 10, 20, 30, 44, 45, 70, 95]


def gop_script():
    """gop = 10 at creation; set_gop(25) before picture 35, IDR requests before 44 and 45 (consecutive) and before 70 (where
    the GOP puts one anyway), set_gop(-1) before 80, a request before 95.  Key pictures: GOP_KEYS."""
    for t in range(120):
        if t == 35:
            yield set_gop(25)
        if t in (44, 45, 70, 95):
            yield request_idr()
        if t == 80:
            yield set_gop(-1)
        yield picture(desktop(W, H, t))


# (src_w, src_h, dst_w, dst_h) of each step and the CSC path it runs
RESIZE_STEPS = [
    (320, 192, 320, 192),       # 1:1, LDG kernel
    (130, 70, 130, 70),         # 1:1 ragged: general kernel, coded 144x80
    (640, 360, 320, 180),       # scaled, tiled, 10 KB of shared memory
    (1920, 1080, 320, 180),     # scaled, tiled, 80 KB: the opt-in tier
    (3840, 2160, 320, 180),     # footprint 307 KB: general kernel
    (160, 96, 320, 192),        # upscale
    (320, 192, 320, 192),       # back to 1:1
]
RESIZE_PICTURES = 4


def resize_script():
    for k, (sw, sh, dw, dh) in enumerate(RESIZE_STEPS):
        if k:
            yield resize(sw, sh, dw, dh)
        for t in range(RESIZE_PICTURES):
            yield picture(desktop(sw, sh, 3 * k + t))


# ---- what each script must reach (checked on the oracle's records by tests/test_longrun_oracle.py, again by the GPU tests) --
def band_deliveries(xs) -> dict:
    """y_start -> number of pictures in which that band was delivered."""
    n = {}
    for x in xs:
        for y0, _ in x.bands:
            n[y0] = n.get(y0, 0) + 1
    return n


def check_fullframe_cqp(xs):
    assert len(xs) >= 512 and [x.index for x in xs if x.is_key] == [0]          # frame_num wraps twice
    paint = [x.index for x in xs if x.qp == FULLFRAME_CQP.paint[1]]
    bursts = [i for i in paint if i - 1 not in paint]
    assert len(bursts) >= 15, bursts                     # paint-over re-armed after every still, scroll and noise alike


def check_striped(xs):
    n = band_deliveries(xs)
    assert n[0] == len(xs) > 256 and n[96] == 1, n       # band 0 wraps frame_num; band 2 is coded once (the IDR)
    assert len(xs) // 7 < n[48] < 256 and len(xs) // 2 < n[144] < 256, n


def check_cbr_pinned(xs):
    T = xs[0].target_bits
    pinned = [x.index for x in xs if x.qp == 51 and x.rc["fullness"] == 64 * T]
    assert len(pinned) >= 50, pinned
    assert any(x.rc["fullness"] <= 0 for x in xs[pinned[-1]:])         # the clamped bucket drains within the script
    assert min(x.qp for x in xs[pinned[-1]:]) < 51


def check_cbr_generous(xs):
    T = xs[0].target_bits
    assert sum(x.qp == 10 for x in xs) >= 50 and sum(x.rc["fullness"] == -4 * T for x in xs) >= 50


def check_cbr_debt(xs):
    assert sum(x.rc["debt"] for x in xs) >= 5 and max(x.qp for x in xs[10:]) < 51


def check_live_cbr(xs):
    """The QP moves after every step, so no step can be ignored on both sides unnoticed."""
    s, qp = LIVE_CBR_STEPS, [x.qp for x in xs]
    assert min(qp[s["up"] + 1: s["up"] + 12]) < qp[s["up"]], qp
    assert max(qp[s["down"] + 1: s["down"] + 12]) > qp[s["down"]], qp
    assert xs[s["idr"]].is_key and xs[s["idr"]].target_bits == int(200 * 1000 / 30)
    assert len({x.target_bits for x in xs[s["remb"]: s["remb"] + 10]}) == 10 and len(set(qp[s["remb"]: s["remb"] + 12])) > 1, qp
    assert max(qp[s["fps60"] + 1: s["fps60"] + 6]) > qp[s["fps60"]], qp
    assert min(qp[s["fps24"] + 1: s["fps24"] + 8]) < qp[s["fps24"]], qp


def check_live_cqp(xs):
    qp = [x.qp for x in xs]
    assert qp[:6] == [30] * 6 and qp[6:12] == [24] * 6 and qp[12:24] == [36] * 12, qp
    assert qp[24:28] == [20] * 4 and qp[28:] == [33] * (len(qp) - 28), qp         # set_qp(33) inside the burst waits for its end


def check_gop(xs):
    assert [x.index for x in xs if x.is_key] == GOP_KEYS
