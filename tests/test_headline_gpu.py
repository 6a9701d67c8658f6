"""GPU parity on the HEADLINE configuration (BASELINE.json configs[2] / [3]), exactly as bench.py drives it.

The reference builds this shape of settings at src/selkies/media_pipeline.py:251-273 (4K capture, CBR, h264_bitrate_kbps,
full frame).  bench.py: 3840x2160 synthetic desktop, CBR 20 Mbit/s @ 60 fps nominal, IDR then P pictures, a 16-picture ring
and the 16-picture scroll cycle — picture 16 is the scroll RESTART, the one picture of the cycle in which nothing is
predictable and every macroblock runs the exhaustive search + refinement.  The pictures go through the same entry point as
the timed legs (b2v_submit_resident, B2V_FLAG_TIMING_CSC, two-stream schedule, several pictures in flight) and every access
unit AND the final reconstruction must equal the oracle's, byte for byte (tests/scenario.py)."""
import dataclasses

import pytest

import oracle
from selkies_b200 import _native as N
from tests import scenario as S
from tests import synth

pytestmark = pytest.mark.gpu

W, H, N_DISTINCT, N_PICS = 3840, 2160, 16, 18
HEADLINE = S.Config(W, H, rc_mode=S.CBR, kbps=20000, fps=60.0, ring_slots=N_DISTINCT, flags=N.B2V_FLAG_TIMING_CSC, entry="resident")


@pytest.fixture(scope="module")
def c2_events():
    oracle.set_threads(0)
    frames = [synth.desktop(W, H, t) for t in range(N_DISTINCT)]
    return [S.picture(frames[i % N_DISTINCT]) for i in range(N_PICS)]


def test_c2_4k_cbr20_idr_plus_17p_bit_exact(c2_events):
    xs = S.pictures(S.run(HEADLINE, c2_events))
    assert [x.is_key for x in xs] == [True] + [False] * (N_PICS - 1)
    # the scroll restart (picture 16) is the expensive one: it must be much larger than a steady scroll picture
    assert len(xs[16].au) > 2 * len(xs[15].au)


def test_c2_4k_striped_8_bands_bit_exact(c2_events):
    rows = -(-(H // 16) // 8)                    # 17 macroblock rows per stripe, as bench.py's striped leg
    S.run(dataclasses.replace(HEADLINE, stripe_rows=rows), c2_events)


def test_c3_second_gpu_same_stream(c2_events):
    """configs[3]: one session per GPU.  A session on device 1 (when the box has one) produces the oracle's stream too."""
    if N.lib().b2v_device_count() < 2:
        pytest.skip("one GPU visible")
    S.run(HEADLINE, c2_events[:6], device=1)
