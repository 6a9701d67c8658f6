"""What a consumer reads from the first slice of an H.264 access unit: the NAL header byte of a droppable picture (B2V_FLAG_DROPPABLE)
and the slice_type of a cut picture (B2V_FLAG_SCENE_CUT), include/b2video.h."""
from __future__ import annotations


def is_droppable(au, offset: int = 0) -> bool:
    """True when the Annex-B access unit starting at `offset` of `au` (bytes or bytearray) is a non-reference picture: the NAL
    header of its first slice (nal_unit_type 1 or 5) carries nal_ref_idc 0.  Anything without a slice NAL (empty, JPEG, parameter
    sets only) is False.  A P picture's first slice follows the first start code, so this reads a few bytes."""
    i = offset
    while True:
        i = au.find(b"\x00\x00\x01", i)
        if i < 0 or i + 3 >= len(au):
            return False
        hdr = au[i + 3]
        if hdr & 0x1F in (1, 5):
            return hdr & 0x60 == 0
        i += 3


def is_intra(au, offset: int = 0) -> bool:
    """True when the first slice of the Annex-B access unit starting at `offset` of `au` is an I slice: slice_type (7.3.3, the second
    ue(v) of the slice header) is 2 or 7.  Every slice of an IDR picture and of a cut picture (B2V_FLAG_SCENE_CUT) is one.  Anything
    without a slice NAL, or whose first slice header ends before its slice_type, is False."""
    i = offset
    while True:
        i = au.find(b"\x00\x00\x01", i)
        if i < 0 or i + 3 >= len(au):
            return False
        if au[i + 3] & 0x1F in (1, 5):
            break
        i += 3
    rbsp, zeros = [], 0
    for b in au[i + 4: i + 16]:               # first_mb_in_slice and slice_type fit in a few bytes; emulation prevention removed
        if zeros >= 2 and b == 3:
            zeros = 0
            continue
        rbsp.append(b)
        zeros = zeros + 1 if b == 0 else 0
    bits = "".join(f"{b:08b}" for b in rbsp)

    def ue(pos):                              # (value, next position), or None when the bits run out
        n = 0
        while pos + n < len(bits) and bits[pos + n] == "0":
            n += 1
        if pos + 2 * n + 1 > len(bits):
            return None
        return int(bits[pos + n: pos + 2 * n + 1], 2) - 1, pos + 2 * n + 1

    first = ue(0)
    slice_type = ue(first[1]) if first else None
    return slice_type is not None and slice_type[0] % 5 == 2
