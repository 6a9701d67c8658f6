"""The picture size cap (B2V_FLAG_SIZE_CAP, include/b2video.h) restated from the syntax reader alone (tests/h264_syntax.py): from a
flag-off stream's macroblocks, the count of every P picture and the QP the rule gives it; from a flagged stream, what a recode kept.
Nothing here reads the oracle or the encoder."""
from __future__ import annotations

from tests import h264_syntax as HS
from tests import h264_syntax_refs as HSR

T = [round(65536 * 2 ** (d / 6)) for d in range(52)]
PCM_MB_TYPE_BITS = 9             # ue(30), the mb_type of I_PCM in a P slice
PCM_SAMPLE_BITS = 384 * 8        # its samples; its pcm_alignment_zero_bits are not counted


def count(pic: HS.Picture) -> int:
    """The count of a P picture: the macroblock_layer() bits of its coded macroblocks, an I_PCM macroblock's without its alignment."""
    return sum(PCM_MB_TYPE_BITS + PCM_SAMPLE_BITS if m.kind == "I_PCM" else m.bits for m in pic.mbs if m.kind != "P_Skip")


def is_capped(pic: HS.Picture) -> bool:
    """P pictures are capped; IDR pictures and scene-cut intra pictures (every macroblock intra) are not."""
    return not pic.idr and any(not m.intra for m in pic.mbs)


def qp_after(bits: int, qp: int, cap: int) -> int:
    if cap <= 0 or qp >= 51 or -(-bits // 8) <= cap:
        return qp
    for d in range(1, 52 - qp):
        if bits <= (8 * cap * T[d]) >> 16:
            return qp + d
    return 51


def decisions(aus, cap: int) -> list:
    """Per picture of a stream coded without the flag (or with cap 0): None when it is not capped, else (count, QP, QP')."""
    out = []
    for pic in HSR.parse_stream(aus):
        if not is_capped(pic):
            out.append(None)
            continue
        bits = count(pic)
        out.append((bits, pic.qp, qp_after(bits, pic.qp, cap)))
    return out


def vectors(pic: HS.Picture) -> list:
    """(vector, ref_idx_l0) of every P_L0_16x16 macroblock of a picture read by h264_syntax_refs; None for I_PCM and P_Skip, whose
    coded syntax does not carry the vector the analysis chose."""
    return [(m.mv, m.ref_idx) if m.kind == "P_L0_16x16" else None for m in pic.mbs]


def mb_kinds(aus) -> list:
    """Per picture, per macroblock: "skip", "pcm" or "coded"."""
    return [["skip" if m.kind == "P_Skip" else "pcm" if m.kind == "I_PCM" else "coded" for m in pic.mbs] for pic in HSR.parse_stream(aus)]
