"""GPU parity of the three-pass P-picture analysis (h264_inter.cu: k_inter_lean, then k_inter_search over the anchor queue and over
the rest) against oracle/h264_ref.c, on the pictures that load each pass differently: the bench stream across two scroll restarts
(the anchor pass runs full searches, the last pass thousands of anchor-vector hits), a still picture (both queues empty), a cut to
noise (almost every macroblock deferred) and the bench stream in striped mode with a clamped anchor group in the last band."""
import dataclasses

import pytest

import oracle
from selkies_b200 import _native as N
from tests import scenario as S
from tests import synth

pytestmark = pytest.mark.gpu

W, H, N_DISTINCT = 3840, 2160, 16
BENCH = S.Config(W, H, rc_mode=S.CBR, kbps=20000, fps=60.0, ring_slots=N_DISTINCT, flags=N.B2V_FLAG_TIMING_CSC, entry="resident")


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


def test_bench_stream_two_scroll_restarts():
    """IDR + 33 P pictures of bench.py's cycle: restarts at pictures 16 and 32, and the pictures after them."""
    frames = [synth.desktop(W, H, t) for t in range(N_DISTINCT)]
    xs = S.pictures(S.run(BENCH, [S.picture(frames[i % N_DISTINCT]) for i in range(34)]))
    assert [x.is_key for x in xs] == [True] + [False] * 33
    assert len(xs[16].au) > 2 * len(xs[15].au) and len(xs[32].au) > 2 * len(xs[31].au)


def test_still_picture():
    """The same picture again and again: every macroblock leaves through the zero vector in the first pass."""
    w, h = 1280, 720
    f = synth.desktop(w, h, 0)
    S.run(dataclasses.replace(BENCH, width=w, height=h, kbps=8000, ring_slots=4), [S.picture(f)] * 5)


@pytest.mark.parametrize("w,h", [(1280, 720), (1304, 744)])
def test_cut_to_noise(w, h):
    """A desktop, then noise: nearly every macroblock fails both early exits and goes to the search passes, the anchors first;
    1304 x 744 also clamps the last column and row of anchor groups."""
    frames = [synth.desktop(w, h, t) for t in range(3)] + [synth.noise(w, h, 40 + t) for t in range(3)]
    S.run(dataclasses.replace(BENCH, width=w, height=h, kbps=8000, ring_slots=4), [S.picture(f) for f in frames])


def test_bench_stream_striped_clamped_anchor_group():
    """8 stripes of 17 macroblock rows at 3840 x 2112 (132 rows): the last band has 13 rows, so its last anchor group has one row
    and its anchor is clamped into it; every other band ends in such a group too.  Pictures 0..17 cover the restart at 16."""
    w, h = 3840, 2112
    rows = -(-(h // 16) // 8)
    assert rows == 17 and (h // 16 - 7 * rows) % 4 == 1
    frames = [synth.desktop(w, h, t) for t in range(N_DISTINCT)]
    S.run(dataclasses.replace(BENCH, width=w, height=h, stripe_rows=rows), [S.picture(frames[i % N_DISTINCT]) for i in range(18)])
