"""The GPU parity cases of the chunked slice assembly (test_slice_chunks_gpu.py) reach the seams they are there for.  The oracle
codes a slice serially, so byte parity says nothing about a branch of k_slice_build that no GPU case runs; these tests parse the
oracle's stream of every case (tests/h264_syntax.py) and find, in the macroblock types of each slice, the placements the case
claims (tests/slice_chunk_cases.py; chunk k of a slice = macroblocks first_mb_in_slice + 256·k onwards).  A change of content or
encoder that moves a case off its seams fails here, without a GPU."""
import pytest

from tests import scenario as S
from tests import slice_chunk_cases as K
from tests.h264_syntax import StreamParser
from tests.slice_chunk_cases import CHUNK


def coded(kind):
    return kind != "P_Skip"


def ue_len(v):
    return 2 * (v + 1).bit_length() - 1


def slice_seams(kinds, idr):
    """The seams one slice reaches, from the types of its macroblocks in order.

    pcm_local0 / pcm_local255   I_PCM at local index 0 / 255 of a chunk k >= 1
    pcm_then_fold               a chunk holding I_PCM, followed by another chunk of the slice
    idr_pcm_chunk1              an IDR slice of more than 256 macroblocks with I_PCM in chunk 1
    one_mb_chunk                the last chunk holds one macroblock
    run_over_chunks             a P_Skip run covering at least two whole chunks, ending in a coded macroblock
    run_into_pcm                the first coded macroblock of a chunk k >= 1 holding I_PCM has a skip run carried from the chunks
                                in front whose ue(v) length differs from that of the chunk's own leading skips
    trailing_run                a trailing skip run of more than 256 macroblocks
    many_chunks                 more than 64 chunks
    many_chunks_pcm             more than 64 chunks and I_PCM in a chunk beyond 32"""
    n = len(kinds)
    chunks = [kinds[i:i + CHUNK] for i in range(0, n, CHUNK)]
    pcm = [k for k, c in enumerate(chunks) if "I_PCM" in c]
    s = set()
    for k in pcm:
        if k >= 1 and chunks[k][0] == "I_PCM":
            s.add("pcm_local0")
        if k >= 1 and len(chunks[k]) == CHUNK and chunks[k][CHUNK - 1] == "I_PCM":
            s.add("pcm_local255")
        if k + 1 < len(chunks):
            s.add("pcm_then_fold")
    if idr and n > CHUNK and 1 in pcm:
        s.add("idr_pcm_chunk1")
    if n % CHUNK == 1:
        s.add("one_mb_chunk")
    if len(chunks) > 64:
        s.add("many_chunks")
        if any(k > 32 for k in pcm):
            s.add("many_chunks_pcm")
    if idr:
        return s
    run_start = 0                                # first macroblock of the skip run open at index i
    for i, kind in enumerate(kinds):
        if not coded(kind):
            continue
        if -(-run_start // CHUNK) + 2 <= i // CHUNK:          # whole chunks ceil(run_start / 256) .. i // 256 - 1
            s.add("run_over_chunks")
        k, local = divmod(i, CHUNK)
        if k >= 1 and k in pcm and run_start < k * CHUNK and all(not coded(t) for t in chunks[k][:local]):
            if ue_len(i - run_start) != ue_len(local):
                s.add("run_into_pcm")
        run_start = i + 1
    if n - run_start > CHUNK:
        s.add("trailing_run")
    return s


def case_seams(case):
    """Every seam reached by a slice of the oracle's stream of `case`."""
    pics = S.pictures(S.run(case.cfg, S.stream(case.frames), gpu=False))
    parsers, seams = {}, set()
    for x in pics:
        for y0, au in x.bands:
            pic = parsers.setdefault(y0, StreamParser()).picture(au)
            for h in pic.headers:
                seams |= slice_seams([m.kind for m in pic.mbs[h["first_mb"]:h["end_mb"]]], pic.idr)
    return seams


@pytest.mark.parametrize("name", sorted(K.CASES))
def test_slice_chunk_case_reaches_its_seams(name):
    case = K.CASES[name]()
    missing = set(case.seams) - case_seams(case)
    assert not missing, f"{name}: the oracle's stream does not reach {sorted(missing)}"


def test_seams_are_found_where_they_are_and_nowhere_else():
    """The finder on hand-made slices: every seam of a slice built to hold it, none in one built to hold none."""
    skip, pcm, p = "P_Skip", "I_PCM", "P_L0_16x16"
    k = [p] + [skip] * (3 * CHUNK - 1) + [pcm] + [skip] * 300
    assert slice_seams(k, False) == {"pcm_local0", "pcm_then_fold", "run_over_chunks", "run_into_pcm", "trailing_run"}
    k = [skip] * (CHUNK - 1) + [pcm] + [skip] * (CHUNK + 1)
    assert slice_seams(k, False) == {"pcm_then_fold", "one_mb_chunk", "trailing_run"}
    k = ["I_16x16"] * CHUNK + [pcm] + ["I_16x16"] * (CHUNK - 2) + [pcm]
    assert slice_seams(k, True) == {"pcm_local0", "pcm_local255", "idr_pcm_chunk1"}
    k = [skip] * (65 * CHUNK) + [pcm]
    assert slice_seams(k, False) == {"many_chunks", "many_chunks_pcm", "one_mb_chunk", "pcm_local0", "run_over_chunks", "run_into_pcm"}
    k = [pcm] + [p] * (2 * CHUNK) + [skip] * (CHUNK - 1)
    assert slice_seams(k, False) == {"pcm_then_fold"}
