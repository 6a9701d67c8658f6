"""The one byte a consumer reads to tell a droppable H.264 access unit (B2V_FLAG_DROPPABLE, include/b2video.h)."""
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
