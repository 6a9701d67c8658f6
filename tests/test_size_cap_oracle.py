"""The picture size cap (B2V_FLAG_SIZE_CAP) in the oracle.  On a scroll restart and the start of a video, with CQP and CBR, droppable
pictures, wide motion, the long-term reference and scene cuts: every picture over the cap is recoded at the QP' of the rule and no
other; pictures up to the first recode are byte-identical to the flag-off stream, and a cap of 0 or one above every picture changes
no byte; QP' <= 51; every stream decodes with libavcodec to the oracle's reconstructions; an I_PCM picture counts its samples; a
recode turns coded macroblocks into P_Skip and back, and I_PCM macroblocks into coded ones.  Prints the largest picture of each content with the flag off and on."""
import numpy as np
import pytest

import oracle
from oracle import avdec
from oracle.cap import SizeCapEncoder
from tests import synth

T = [round(65536 * 2 ** (d / 6)) for d in range(52)]


def rule(bits, qp, cap):
    """include/b2video.h B2V_FLAG_SIZE_CAP, stated again: the QP a P picture of `bits` is coded at."""
    if cap <= 0 or qp >= 51 or -(-bits // 8) <= cap:
        return qp
    for d in range(1, 52 - qp):
        if bits <= (8 * cap * T[d]) >> 16:
            return qp + d
    return 51


def scroll_restart(w, h):
    """A still desktop, then its text region scrolls 8 px per picture."""
    return [synth.desktop(w, h, 0)] * 3 + [synth.desktop(w, h, t) for t in range(1, 5)]


def video_start(w, h):
    """A still desktop, then every picture new content (noise), then still again."""
    return [synth.desktop(w, h)] * 2 + [synth.noise(w, h, k) for k in range(3)] + [synth.noise(w, h, 2)]


CONTENTS = {"scroll_restart": scroll_restart, "video_start": video_start}


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


def _encode(frames, cap, wide=False, ltr=False, droppable=False, cut=False, on=True, **kw):
    h, w = frames[0].shape[:2]
    e = SizeCapEncoder(w, h)
    e.set_droppable(droppable)
    e.set_wide_motion(wide)
    e.set_long_term_ref(ltr)
    if on:
        e.set_size_cap(True, cut)
        e.max_picture_bytes = cap
    elif cut:
        e.set_scene_cut(True)
    aus, recs, states = [], [], []
    for i, f in enumerate(frames):
        aus.append(e.encode_bgra(f, i == 0, **kw))
        recs.append(e.recon())
        states.append(e.cap_state() if on else None)
    e.close()
    return aus, recs, states


def _assert_decodes(aus, recs, w, h):
    dec = avdec.decode_stream(aus, quiet=True)
    assert len(dec) == len(aus)
    for k, ((Y, U, V), (ry, ruv)) in enumerate(zip(dec, recs)):
        assert np.array_equal(Y, ry[:h, :w]), f"picture {k}: decoded luma != reconstruction"
        assert np.array_equal(U, ruv[:h // 2, 0:w:2]) and np.array_equal(V, ruv[:h // 2, 1:w:2]), f"picture {k}: chroma"


def _check(frames, cap, **kw):
    """The capped stream against the flag-off stream and the rule; returns the capped stream's states."""
    h, w = frames[0].shape[:2]
    off, _, _ = _encode(frames, 0, on=False, **kw)
    aus, recs, st = _encode(frames, cap, **kw)
    _assert_decodes(aus, recs, w, h)
    first = next((k for k, s in enumerate(st) if s["recoded"]), len(frames))
    assert aus[:first] == off[:first]
    for k, s in enumerate(st):
        assert s["qp_final"] <= 51
        if k == 0 or s["bits"] == 0:          # the IDR picture, cut pictures: not capped
            assert not s["recoded"]
            continue
        assert s["qp_final"] == rule(s["bits"], s["qp"], cap), (k, s)
        assert s["recoded"] == (s["qp_final"] != s["qp"])
    return aus, recs, st


@pytest.mark.parametrize("name", list(CONTENTS))
@pytest.mark.parametrize("opts", [dict(), dict(wide=True), dict(droppable=True), dict(ltr=True, cut=True),
                                  dict(rc_mode=0, target_bits=60000)])
def test_recodes_follow_the_rule(name, opts):
    frames = CONTENTS[name](320, 192)
    _, _, zero = _encode(frames, 0, **opts)
    p_bytes = sorted(-(-s["bits"] // 8) for s in zero[1:] if s["bits"])
    cap = max(1, p_bytes[-1] // 2)          # half the largest P picture: at least that one is recoded
    _, _, st = _check(frames, cap, **opts)
    assert any(s["recoded"] for s in st), (name, opts)


@pytest.mark.parametrize("name", list(CONTENTS))
def test_no_cap_changes_no_byte(name):
    frames = CONTENTS[name](320, 192)
    off, _, _ = _encode(frames, 0, on=False)
    for cap in (0, 1 << 30):
        aus, _, st = _encode(frames, cap)
        assert aus == off and not any(s["recoded"] for s in st)



def kinds_contents(w, h):
    """Pictures whose recode changes macroblock kinds, with the QP and the cap that recode them: (name, frames, qp, cap).
      mild:  a desktop, then the same with +-3 of noise: zero vectors with a small residual at QP 16, none at QP' (coded -> P_Skip);
      grid:  the desktop, then noise with the desktop kept in every third macroblock of every other row: at QP 10 the noise is I_PCM
             and the kept macroblocks, whose three neighbours are all I_PCM, are P_Skip at the zero vector; at QP' the noise is coded
             with the vectors the analysis found, which the kept macroblocks' predictor now reads (I_PCM -> coded, P_Skip -> coded);
      noise: the desktop, then noise: every macroblock I_PCM at QP 10, a 92 KB picture at 320x192 under a 20 000-byte cap."""
    base = synth.desktop(w, h)
    mild = base.copy()
    mild[..., :3] = np.clip(base[..., :3].astype(int) + np.random.default_rng(5).integers(-3, 4, size=(h, w, 1)), 0, 255)
    grid = synth.noise(w, h, 3).copy()
    for y in range(1, h // 16, 2):
        for x in range(1, w // 16, 3):
            grid[y * 16:y * 16 + 16, x * 16:x * 16 + 16] = base[y * 16:y * 16 + 16, x * 16:x * 16 + 16]
    scale = w * h / (320 * 192)
    return [("mild", [base, mild], 16, int(300 * scale)), ("grid", [base, grid], 10, int(20000 * scale)),
            ("noise", [base, synth.noise(w, h, 0)], 10, int(20000 * scale))]


def test_recode_changes_macroblock_kinds():
    """P_Skip both ways and I_PCM -> coded, as the independent reader finds them, each on a picture the rule recoded.  A recode never
    turns a coded macroblock into I_PCM on these contents: a coarser QP does not lengthen a macroblock's levels (DESIGN.md §5.15)."""
    from tests import h264_model_size_cap as M
    changes = {}
    for name, frames, qp, cap in kinds_contents(320, 192):
        off, _, _ = _encode(frames, 0, on=False, qp=qp)
        aus, _, st = _check(frames, cap, qp=qp)
        assert st[1]["recoded"], name
        a, b = M.mb_kinds(off), M.mb_kinds(aus)
        for x, y in zip(a[1], b[1]):
            if x != y:
                changes.setdefault((x, y), name)
    assert {("coded", "skip"), ("skip", "coded"), ("pcm", "coded")} <= set(changes), changes


def test_pcm_picture_is_counted_whole():
    """A P picture of I_PCM macroblocks counts their samples: 320x192 noise at QP 10 is 92 KB, over a 20 000-byte cap, and recoded."""
    frames = [synth.desktop(320, 192), synth.noise(320, 192, 0)]
    aus, _, st = _encode(frames, 20000, qp=10)
    assert st[1]["bits"] >= 240 * 384 * 8 and st[1]["recoded"] and st[1]["qp_final"] > 10
    assert len(aus[1]) < len(_encode(frames, 0, on=False, qp=10)[0][1])


def test_largest_picture_table(capsys):
    """The largest picture of each content at 1280x720, CQP 22, with the flag off and with a cap of 8 000 bytes."""
    rows = []
    for name, make in CONTENTS.items():
        frames = make(1280, 720)
        off, _, _ = _encode(frames, 0, on=False, qp=22)
        aus, _, st = _encode(frames, 8000, qp=22)
        rows.append((name, max(len(a) for a in off[1:]), max(len(a) for a in aus[1:]), sum(s["recoded"] for s in st)))
    with capsys.disabled():
        print("\ncontent          largest P, off   largest P, cap 8000   recoded")
        for r in rows:
            print(f"{r[0]:<16} {r[1]:>15} {r[2]:>22} {r[3]:>9}")
