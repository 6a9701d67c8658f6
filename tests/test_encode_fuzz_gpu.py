"""Randomised parity: CUDA encoder vs oracle over random sizes, slice layouts, QPs / bitrates, IDR positions and
content mixes (edge cases: one-macroblock-wide pictures, cropped sizes, search windows clamped at every picture edge)."""
import numpy as np
import pytest

from tests import scenario as S
from tests import synth

pytestmark = pytest.mark.gpu


def make_frames(rng, w, h, n):
    kind = rng.integers(0, 5)
    base = synth.noise(w, h, int(rng.integers(0, 1000)))
    out = []
    for t in range(n):
        if kind == 0:
            f = synth.desktop(w, h, t)
        elif kind == 1:
            f = synth.gradient(w, h, t)
        elif kind == 2:
            f = np.roll(base, (int(rng.integers(-20, 21)) * t, int(rng.integers(-20, 21)) * t), axis=(0, 1))
        elif kind == 3:
            f = synth.bars(w, h, t)
        else:   # mixed: half smooth, half noise, moving split line
            f = synth.gradient(w, h, t).copy()
            cut = (h // 2 + 4 * t) % h
            f[:cut] = base[:cut]
        out.append(np.ascontiguousarray(f))
    return out


@pytest.mark.parametrize("seed", range(24))
def test_random_configuration(seed):
    rng = np.random.default_rng(1000 + seed)
    w = int(rng.choice([16, 18, 32, 48, 66, 130, 160, 258, 322, 400])) & ~1
    h = int(rng.choice([16, 18, 34, 48, 70, 96, 130, 176, 226])) & ~1
    n = int(rng.integers(2, 6))
    slice_rows = int(rng.choice([1, 1, 2, 3, 100]))
    frames = make_frames(rng, w, h, n)
    idr_at = tuple(sorted({0} | {int(i) for i in rng.integers(1, n, size=int(rng.integers(0, 2)))}))
    if rng.integers(0, 3) == 0:
        cfg = S.Config(w, h, rc_mode=S.CBR, kbps=int(rng.choice([100, 400, 2000, 20000])), fps=30.0, slice_rows=slice_rows)
    else:
        cfg = S.Config(w, h, qp=int(rng.choice([0, 8, 18, 24, 30, 37, 45, 51])), slice_rows=slice_rows)
    S.run(cfg, S.stream(frames, idr_at))


@pytest.mark.parametrize("seed", range(12))
def test_random_striped_configuration(seed):
    """Same, in striped mode (random band height) with paint-over switched on in the constant-QP runs and still pictures mixed in."""
    rng = np.random.default_rng(5000 + seed)
    w = int(rng.choice([32, 66, 130, 160, 258, 322])) & ~1
    h = int(rng.choice([48, 70, 96, 130, 176, 226])) & ~1
    n = int(rng.integers(3, 8))
    slice_rows = int(rng.choice([1, 1, 2]))
    mbh = (h + 15) // 16
    stripe_rows = slice_rows * int(rng.integers(1, max(2, mbh // slice_rows)))
    frames = make_frames(rng, w, h, n)
    for t in range(1, n):
        if rng.integers(0, 3) == 0:
            frames[t] = frames[t - 1]                         # a still picture: every band is dropped
        else:
            frames[t][: h // 3] = frames[0][: h // 3]         # static top third
    idr_at = tuple(sorted({0} | {int(i) for i in rng.integers(1, n, size=int(rng.integers(0, 2)))}))
    layout = dict(stripe_rows=stripe_rows, slice_rows=slice_rows)
    if rng.integers(0, 3) == 0:
        cfg = S.Config(w, h, rc_mode=S.CBR, kbps=int(rng.choice([200, 1500, 20000])), fps=30.0, **layout)
    else:
        cfg = S.Config(w, h, qp=int(rng.choice([10, 24, 30, 38, 47])), paint=(int(rng.integers(1, 3)), int(rng.choice([8, 16, 22])), 1), **layout)
    S.run(cfg, S.stream(frames, idr_at))
