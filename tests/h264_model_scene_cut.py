"""Scene cuts (B2V_FLAG_SCENE_CUT, DESIGN.md §5.14) in the independent decisions model: the intra estimate, the cost of the vectors
tests/h264_model.py predicts, and the rule.  Built on that model alone (prediction, motion cost, the lean pass's exits and the search
decisions); nothing here comes from oracle/ or selkies_b200/.

For a P picture, from the source luma, the reconstruction of its short-term reference, the long-term picture's (None while there is
none), the previous picture's parsed records and, with wide motion, the decimated luma of the picture and of its reference:
  cost_inter(mb) = the luma cost of the prediction decide() chooses (refIdx 1: the long-term picture at the zero vector) —
                   motion_cost(SAD, mv), 0 when the SAD is at most 96·λ; while there is a long-term picture, the smaller of that and
                   the same cost of its zero vector;
  cost_intra(mb) = the smallest SAD of Intra16x16 vertical, horizontal and DC prediction (8.3.3) from the source's neighbours,
                   available inside the picture, + 16·λ;
  cut ⇔ Σ cost_intra < Σ cost_inter."""
from __future__ import annotations

import numpy as np

from tests import h264_model as M

INTRA_MB_BITS = 16


def intra_estimate(y, mbx, mby):
    """8.3.3 Intra16x16 vertical, horizontal and DC of the macroblock from the source luma `y` itself: the smallest SAD."""
    x0, y0 = 16 * mbx, 16 * mby
    blk = y[y0:y0 + 16, x0:x0 + 16]
    top = y[y0 - 1, x0:x0 + 16] if mby > 0 else None
    left = y[y0:y0 + 16, x0 - 1] if mbx > 0 else None
    if top is not None and left is not None:
        dc = (int(top.sum()) + int(left.sum()) + 16) >> 5
    elif top is not None:
        dc = (int(top.sum()) + 8) >> 4
    elif left is not None:
        dc = (int(left.sum()) + 8) >> 4
    else:
        dc = 128
    costs = [M.sad(blk, np.full((16, 16), dc))]
    if top is not None:
        costs.append(M.sad(blk, np.broadcast_to(top[None, :], (16, 16))))
    if left is not None:
        costs.append(M.sad(blk, np.broadcast_to(left[:, None], (16, 16))))
    return min(costs)


def inter_cost(blk, ref, lt, d: M.Decision, x0, y0, qp):
    thr = M.EARLY_SAD_PER_LAMBDA * M.LAMBDA[qp]

    def cost(s, mv):
        return 0 if s <= thr else M.motion_cost(s, mv, qp)
    if d.ref_idx == 1:
        c = cost(M.sad(blk, M.full_pred(lt, x0, y0, (0, 0))), (0, 0))
    else:
        c = cost(M.sad(blk, M.luma_inter(ref, x0, y0, d.mv)), d.mv)
    if lt is not None:
        c = min(c, cost(M.sad(blk, M.full_pred(lt, x0, y0, (0, 0))), (0, 0)))
    return c


def picture_costs(src_y, ref, lt, prev_mbs, qp, wide=False, dec=None, dist=(1, 1)):
    """(Σ cost_intra, Σ cost_inter) of a P picture.  prev_mbs: the previous picture's parsed records by address.  dec: (decimated
    luma of this picture's source, of its reference's), wide motion only.  Anchors are decided first, then the rest."""
    h, w = src_y.shape
    mbw, mbh = w // 16, h // 16
    y = np.asarray(src_y, np.int64)
    ref, lt = np.asarray(ref, np.int64), None if lt is None else np.asarray(lt, np.int64)
    order = sorted(range(mbw * mbh), key=lambda a: M.anchor_of(a % mbw, a // mbw, mbw, 0, mbh) != (a % mbw, a // mbw))
    decided, intra, inter = {}, 0, 0
    for a in order:
        mbx, mby = a % mbw, a // mbw
        x0, y0 = 16 * mbx, 16 * mby
        blk = y[y0:y0 + 16, x0:x0 + 16]
        anchor = M.anchor_of(mbx, mby, mbw, 0, mbh)
        is_anchor = anchor == (mbx, mby)
        coarse = None
        if wide and is_anchor:
            coarse = M.coarse_search(dec[0], dec[1], mbx, mby, mbw, 0, mbh, M.sad(blk, ref[y0:y0 + 16, x0:x0 + 16]), qp)
        d = M.decide(blk, ref, lt, prev_mbs[a], x0, y0, qp, wide, dist, None if is_anchor else decided[anchor], coarse)
        decided[(mbx, mby)] = d
        inter += inter_cost(blk, ref, lt, d, x0, y0, qp)
        intra += intra_estimate(y, mbx, mby) + INTRA_MB_BITS * M.LAMBDA[qp]
    return intra, inter


def cuts(intra, inter):
    """§5.14: the picture is coded as an intra picture."""
    return intra < inter
