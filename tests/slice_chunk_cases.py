"""The streams of test_slice_chunks_gpu.py, shared with test_slice_chunks_oracle.py, which checks on the oracle's bytes that each
reaches the seams of the chunked slice assembly it is there for.

k_slice_build (selkies_b200/csrc/h264_entropy.cu, DESIGN.md §5.5) builds a slice in chunks of CHUNK macroblocks, one block per
chunk: chunk k of a slice holds the macroblocks first_mb_in_slice + CHUNK·k .. first_mb_in_slice + CHUNK·k + CHUNK - 1 (addresses
relative to the band in striped mode, as first_mb_in_slice is).  The pictures are flat grey with tiles of noise, which are
I_PCM at QP 0, and lightly changed tiles, which are coded in a few bits (synth.tiles); everything else is P_Skip."""
from dataclasses import dataclass

from tests import scenario as S
from tests import synth

CHUNK = 256


@dataclass
class Case:
    cfg: S.Config
    frames: list
    seams: tuple                 # what test_slice_chunks_oracle.py must find in the oracle's stream (see its `slice_seams`)


def seams_1024(qp):
    """1024x272 in one P slice of 1088 macroblocks (5 chunks, the last of 64).  Picture 1: I_PCM at local 255 of chunk 0, 0 and 255
    of chunk 1, 0 of chunk 2, inside chunk 2 and as the slice's last macroblock, coded macroblocks in chunks 0 and 3, so that
    chunks without I_PCM sit between chunks with it.  Picture 2 is still: one skip run over all five chunks.  Picture 3: I_PCM in
    chunk 0, then a run over the whole of chunks 1 and 2 into I_PCM at local 0 of chunk 3, then a trailing run of 319.
    Picture 4: a coded macroblock in chunk 1, then a run over chunks 2 and 3 into I_PCM at local 0 of chunk 4."""
    w, h = 1024, 272
    f0 = synth.tiles(w, h)
    f1 = synth.tiles(w, h, (255, 256, 511, 512, 700, 1087), (100, 900), seed=1)
    f3 = synth.tiles(w, h, (200, 768), seed=3, base=f1)
    f4 = synth.tiles(w, h, (1024,), (300,), seed=4, base=f3)
    return Case(S.Config(w, h, qp=qp, slice_rows=100), [f0, f1, f1, f3, f4],
                ("pcm_local0", "pcm_local255", "pcm_then_fold", "run_over_chunks", "run_into_pcm", "trailing_run"))


def one_mb_tail():
    """4112x32 (257 macroblocks per row): IDR and P slices of one row, 257 macroblocks, whose last chunk holds one macroblock.
    IDR: I_PCM at 0, 255, 256 (the one-macroblock chunk) of row 0, inside row 1 and at its one-macroblock chunk.  P: I_PCM at
    0, 255 and 256 of row 0 and at the two seams of row 1; then a skip run over the whole of chunk 0 into I_PCM in the
    one-macroblock chunk; then a still picture (trailing runs of 257)."""
    w, h = 4112, 32
    f0 = synth.tiles(w, h, (0, 255, 256, 300, 513))
    f1 = synth.tiles(w, h, (0, 255, 256, 512, 513), seed=1, base=f0)
    f2 = synth.tiles(w, h, (256,), seed=2, base=f1)
    return Case(S.Config(w, h, qp=0, slice_rows=1, idr_slice_mbs=257), [f0, f1, f2, f2],
                ("pcm_local0", "pcm_then_fold", "idr_pcm_chunk1", "one_mb_chunk", "run_into_pcm", "trailing_run"))


def wide_idr():
    """7680x48: IDR slices of a whole row, 480 macroblocks (chunks of 256 + 224), I_PCM at the seam of every row; then one P slice
    of 1440 macroblocks (6 chunks) with I_PCM at the seam of chunks 2 / 3 and at local 0 of chunk 5."""
    w, h = 7680, 48
    f0 = synth.tiles(w, h, (255, 256, 735, 736, 1216))
    f1 = synth.tiles(w, h, (767, 768, 1280), (100,), seed=1, base=f0)
    return Case(S.Config(w, h, qp=0, idr_slice_mbs=480), [f0, f1],
                ("pcm_local0", "pcm_local255", "pcm_then_fold", "idr_pcm_chunk1"))


def whole_4k_desktop():
    """3840x2160 in one slice of 32400 macroblocks (127 chunks), desktop content under the CBR controller: scroll pictures whose
    every chunk holds coded macroblocks (more than 32 aggregates in front of most chunks), and a still picture whose one skip run
    crosses all 127 chunks."""
    w, h = 3840, 2160
    frames = [synth.desktop(w, h, t) for t in (0, 1, 2, 2, 3)]
    return Case(S.Config(w, h, rc_mode=S.CBR, kbps=20000, fps=60.0, slice_rows=135), frames, ("many_chunks", "trailing_run"))


def whole_4k_pcm(cbr=False):
    """3840x2160 in one slice of 32400 macroblocks (127 chunks) at QP 0.  Picture 1: I_PCM at the seams of chunks 31 / 32 / 33, at
    local 0 of chunks 64 and 126 and as the last macroblock, coded macroblocks in chunks 0, 40 and 100.  Picture 2 is still.
    Picture 3: I_PCM in chunk 0, then a skip run over the 63 chunks 1..63 into I_PCM at local 0 of chunk 64, then one over
    chunks 65..125 into I_PCM at local 0 of chunk 126.  Picture 4: I_PCM in chunk 33, a coded macroblock in chunk 100 and a
    trailing run of over 6000.
    cbr: the same pictures under the CBR controller, each after three still ones (a paint-over burst at QP 0 codes the tiles as
    I_PCM): the controller's bit count of every picture that holds I_PCM includes the raw samples."""
    w, h = 3840, 2160
    c = CHUNK
    f0 = synth.tiles(w, h)
    f1 = synth.tiles(w, h, (31 * c, 32 * c - 1, 32 * c, 33 * c - 1, 33 * c, 64 * c, 126 * c, 32399), (10, 40 * c + 7, 100 * c + 100), seed=1)
    f3 = synth.tiles(w, h, (5, 64 * c, 126 * c), seed=3, base=f1)
    f4 = synth.tiles(w, h, (33 * c + 17,), (100 * c + 100,), seed=4, base=f3)
    seams = ("pcm_local0", "pcm_local255", "pcm_then_fold", "run_over_chunks", "run_into_pcm", "trailing_run", "many_chunks_pcm")
    if cbr:
        return Case(S.Config(w, h, rc_mode=S.CBR, kbps=20000, fps=60.0, slice_rows=135, paint=(2, 0, 4)), [f0] * 4 + [f1, f1, f3, f4],
                    seams)
    return Case(S.Config(w, h, qp=0, slice_rows=135), [f0, f1, f1, f3, f4], seams)


def striped_4k():
    """3840x2112 in bands of 17 rows (4080 macroblocks, 16 chunks; the last band 13 rows, 3120 macroblocks, 13 chunks), one slice
    per band: I_PCM at chunk seams inside band 0 and inside the last band, whose first_mb_in_slice and chunk boundaries are
    relative to the band."""
    w, h = 3840, 2112
    c, last = CHUNK, 7 * 17 * 240
    f0 = synth.tiles(w, h)
    f1 = synth.tiles(w, h, (c - 1, c, 15 * c - 1, 4079, last + c - 1, last + c, last + 12 * c), (3000, last + 1000), seed=1)
    f2 = synth.tiles(w, h, (7, 8 * c, last + 8 * c), seed=2, base=f1)
    return Case(S.Config(w, h, qp=0, stripe_rows=17), [f0, f1, f2],
                ("pcm_local0", "pcm_local255", "pcm_then_fold", "run_over_chunks", "run_into_pcm", "trailing_run"))


CASES = {
    "seams_1024_qp0": lambda: seams_1024(0),
    "seams_1024_qp4": lambda: seams_1024(4),
    "one_mb_tail": one_mb_tail,
    "wide_idr": wide_idr,
    "whole_4k_desktop": whole_4k_desktop,
    "whole_4k_pcm": whole_4k_pcm,
    "whole_4k_pcm_cbr": lambda: whole_4k_pcm(cbr=True),
    "striped_4k": striped_4k,
}
