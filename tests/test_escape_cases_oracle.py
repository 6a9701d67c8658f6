"""The GPU parity cases that cover the escape step at its boundaries reach them.  The device copies a segment 16 bytes per thread,
4096 bytes per round (copy_escaped in selkies_b200/csrc/bitstream.cuh); these tests compute, from the oracle's bytes, where the
escapes of each case sit, so that a change of content or encoder that moves them away from the boundaries fails without a GPU.

- H.264 (test_encode_gpu.py::test_escape_boundaries_bit_exact): emulation-prevention bytes in front of RBSP bytes i with
  i mod 16 in {0, 1} (the zero run in front of them starts in the previous thread's chunk) and past byte 4096 of their slice.
- JPEG (test_jpeg_gpu.py::test_jpeg_stripes_bit_exact at 640x96, one stripe, quality 92): FF bytes at scan offsets = 15 mod 16
  (the stuffed 00 shifts the next thread's bytes) and past byte 4096."""
import numpy as np

import oracle
from tests import scenario as S
from tests import synth


def h264_escape_positions(au: bytes) -> list:
    """RBSP position of the byte behind every emulation-prevention byte of the slice NAL units of an Annex B access unit."""
    pos = []
    for nal in au.split(b"\x00\x00\x01")[1:]:
        nal = nal.rstrip(b"\x00")                  # the leading zero of the next 4-byte start code
        if nal[0] & 31 not in (1, 5):
            continue
        z = r = 0
        for b in nal[1:]:
            if z >= 2 and b == 3:
                pos.append(r)
                z = 0
                continue
            z = z + 1 if b == 0 else 0
            r += 1
    return pos


def jpeg_ff_positions(jfif: bytes) -> list:
    """Offset, in the unstuffed entropy-coded data, of every FF byte of a baseline JFIF file with one scan."""
    k = jfif.index(b"\xff\xda")
    scan = jfif[k + 2 + int.from_bytes(jfif[k + 2:k + 4], "big"):]
    assert scan[-2:] == b"\xff\xd9"
    scan = scan[:-2]
    pos, i, r = [], 0, 0
    while i < len(scan):
        if scan[i] == 0xFF:
            assert scan[i + 1] == 0
            pos.append(r)
            i += 1
        i += 1
        r += 1
    return pos


def test_escape_cases_reach_the_copy_boundaries():
    w, h = 1280, 720
    enc = oracle.RefEncoder(w, h, 0)
    ep = []
    for t in range(3):
        ep += h264_escape_positions(enc.encode_bgra(synth.desktop(w, h, t), t == 0, rc_mode=S.CQP, qp=10))
    assert any(r % 16 in (0, 1) for r in ep), ep
    assert any(r >= 4096 for r in ep), ep
    ff = jpeg_ff_positions(oracle.jpeg_encode_bgra(np.ascontiguousarray(synth.desktop(640, 96, 1)), 92))
    assert any(r % 16 == 15 for r in ff), ff
    assert any(r >= 4096 for r in ff), ff
