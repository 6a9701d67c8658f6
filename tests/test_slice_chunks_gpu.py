"""GPU parity of the chunked slice assembly (k_slice_build, DESIGN.md §5.5) at the seams no other test reaches: I_PCM beyond
the first chunk of a slice (a successor waits for the inclusive state of a chunk holding I_PCM, and the byte-alignment walk
starts from a carried bit position and skip run), IDR slices of more than 256 macroblocks, a last chunk of one macroblock,
skip runs carried over wholly skipped chunks, and slices of 127 chunks (the look-back's second round of 32).  The streams are
in tests/slice_chunk_cases.py; test_slice_chunks_oracle.py checks on the oracle's bytes that each reaches its seams.  Every
case goes through tests/scenario.py: bytes, QP, key flag, reconstruction and the libavcodec decode."""
import pytest

from tests import scenario as S
from tests import slice_chunk_cases as K

pytestmark = pytest.mark.gpu


def run(name):
    case = K.CASES[name]()
    xs = S.pictures(S.run(case.cfg, S.stream(case.frames)))
    assert [x.is_key for x in xs] == [True] + [False] * (len(case.frames) - 1)
    return xs


@pytest.mark.parametrize("qp", [0, 4])
def test_pcm_at_chunk_seams(qp):
    """One P slice of 5 chunks: I_PCM at both ends of chunk 1 and around it, ordinary coded chunks between chunks with I_PCM,
    a still picture, skip runs over two whole chunks into I_PCM at local index 0."""
    run(f"seams_1024_qp{qp}")


def test_last_chunk_of_one_macroblock():
    """IDR and P slices of 257 macroblocks: I_PCM in the one-macroblock chunk, of the IDR (no mb_skip_run) and after a run over
    the whole of chunk 0; trailing runs of 257."""
    run("one_mb_tail")


def test_idr_slices_longer_than_a_chunk():
    """7680x48 with IDR slices of a whole row (480 macroblocks: chunks of 256 + 224), I_PCM at every row's seam."""
    run("wide_idr")


def test_whole_picture_slice_4k_desktop():
    """One 4K slice of 127 chunks on desktop content under the CBR controller: most chunks have more than 32 chunks in front of
    them, and the still picture's skip run crosses all of them."""
    run("whole_4k_desktop")


@pytest.mark.parametrize("rc", ["cqp", "cbr"])
def test_whole_picture_slice_4k_pcm(rc):
    """One 4K slice of 127 chunks at QP 0: I_PCM at the seams of chunks 31 / 32 / 33 and at local index 0 of chunks 64 and 126
    behind skip runs over 63 and 61 wholly skipped chunks.  cbr: the same pictures in a paint-over burst at QP 0 under the CBR
    controller, whose bit count of those pictures includes the raw samples."""
    xs = run("whole_4k_pcm_cbr" if rc == "cbr" else "whole_4k_pcm")
    if rc == "cbr":
        assert [x.qp for x in xs][4:] == [0] * 4 and xs[3].qp > 0


def test_striped_band_relative_chunks():
    """3840x2112 in bands of 17 rows, one slice per band (16 chunks; the last band 13): I_PCM at chunk seams of band 0 and of the
    last band, whose chunk boundaries count from the band's first macroblock."""
    run("striped_4k")
