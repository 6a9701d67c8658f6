"""The comparator of tests/scenario.py, without a GPU: records shaped like the session's output, built from the oracle's, pass;
each kind of disagreement the GPU could produce fails."""
import struct

import pytest

from selkies_b200.session import EncodedFrame
from tests import scenario as S
from tests import synth

LAYOUTS = {"fullframe": S.Config(64, 48), "striped": S.Config(64, 80, stripe_rows=2),
           "pixelflux": S.Config(64, 80, stripe_rows=2, header_mode=S.HDR_PIXELFLUX)}
MUTATIONS = {"byte": lambda g: setattr(g, "data", g.data[:-1] + bytes([g.data[-1] ^ 1])),
             "qp": lambda g: setattr(g, "qp", g.qp + 1),
             "is_key": lambda g: setattr(g, "is_key", not g.is_key),
             "height": lambda g: setattr(g, "height", g.height - 1),
             "header": lambda g: setattr(g, "data", g.data[:3] + bytes([g.data[3] ^ 1]) + g.data[4:])}


def session_output(cfg, seg):
    """What the session delivers for the oracle's pictures: one record per band, behind the 10-byte header in pixelflux mode."""
    got = []
    for x in seg.pictures:
        for y0, au in x.bands:
            bh = min(cfg.height - y0, cfg.stripe_rows * 16) if cfg.stripe_rows else cfg.height
            hdr = struct.pack(">BBHHHH", 4, x.is_key, x.index, y0, cfg.width, bh) if cfg.header_mode == S.HDR_PIXELFLUX else b""
            got.append(EncodedFrame(hdr + au, x.index, x.is_key, x.qp, 0, 0, y0, bh))
    return got


@pytest.mark.parametrize("layout", LAYOUTS)
def test_check_segment_accepts_the_oracle_and_rejects_one_change(layout):
    cfg = LAYOUTS[layout]
    o = S.OracleSide(cfg)
    seg = S.Segment((cfg.width, cfg.height), 0, [o.picture(synth.desktop(cfg.width, cfg.height, t), "start") for t in range(3)])
    rec = o.enc.recon()
    S._check_segment(cfg, seg, session_output(cfg, seg), rec, rec, decode=True)
    for name, mutate in MUTATIONS.items():
        if name == "header" and cfg.header_mode != S.HDR_PIXELFLUX:
            continue
        got = session_output(cfg, seg)
        mutate(got[-1])
        with pytest.raises(AssertionError):
            S._check_segment(cfg, seg, got, rec, rec, decode=False)
