"""Pins oracle/h264_ref.c against an independent decoder: every access unit decodes with libavcodec's
h264 decoder and the decoded planes equal the encoder's own reconstruction bit-for-bit (SURVEY.md §8c.4)."""
import numpy as np
import pytest

import oracle
from oracle import avdec
from tests import synth


def split_nals(au: bytes):
    """Annex-B splitter following the reference's _split_bitstream (webrtc/codecs/h264.py:238-263)."""
    out, i = [], 0
    while True:
        i = au.find(b"\x00\x00\x01", i)
        if i < 0:
            break
        i += 3
        j = au.find(b"\x00\x00\x01", i)
        if j < 0:
            out.append(au[i:])
            break
        end = j - 1 if au[j - 1] == 0 else j
        out.append(au[i:end])
    return out


def run(w, h, frames, qp, slice_rows=1, idr_at=(0,)):
    enc = oracle.RefEncoder(w, h, slice_rows)
    aus, recs = [], []
    for i, f in enumerate(frames):
        aus.append(enc.encode_bgra(f, i in idr_at, qp=qp))
        recs.append(enc.recon())
    dec = avdec.decode_stream(aus, quiet=True)
    assert len(dec) == len(frames)
    for (Y, U, V), (ry, ruv) in zip(dec, recs):
        assert np.array_equal(Y, ry[:h, :w])
        assert np.array_equal(U, ruv[: h // 2, 0:w:2])
        assert np.array_equal(V, ruv[: h // 2, 1:w:2])
    return aus, dec


@pytest.mark.parametrize("qp", [0, 10, 22, 30, 40, 51])
def test_noise_all_qps(qp):
    run(64, 48, [synth.noise(64, 48, 1), synth.noise(64, 48, 2)], qp)


@pytest.mark.parametrize("slice_rows", [1, 2, 3, 100])
def test_slicing(slice_rows):
    run(160, 96, [synth.desktop(160, 96, t) for t in range(4)], 28, slice_rows)
    run(96, 80, [synth.bars(96, 80, t) for t in range(4)], 26, slice_rows)


def test_default_slicing_decodes_and_saves_bits():
    """slice_rows = 0: P pictures in 8-row slices (P_Skip infers moving vectors inside a slice), IDR pictures in sub-row slices /
    one slice per row.  A scrolling picture must cost clearly less than with one row per slice, and the key frame the same."""
    w, h = 640, 368                                                       # 23 macroblock rows: slices of 8, 8, 7
    frames = [synth.desktop(w, h, t) for t in range(5)]
    a8, _ = run(w, h, frames, 30, 0, idr_at=(0, 3))
    a1, _ = run(w, h, frames, 30, 1, idr_at=(0, 3))
    assert len(a8[0]) == len(a1[0]) and len(a8[3]) == len(a1[3])          # IDR slicing does not depend on slice_rows
    assert sum(len(a8[i]) for i in (1, 2, 4)) < 0.9 * sum(len(a1[i]) for i in (1, 2, 4))
    n_p_slices = sum(1 for n in split_nals(a8[1]) if (n[0] & 31) == 1)
    assert n_p_slices == 3
    run(1280, 720, [synth.desktop(1280, 720, t) for t in range(3)], 33, 0)   # 45 rows, IDR in two segments per row


def test_negative_idr_slice_mbs_is_rejected():
    """IDR slices never span rows: a negative idr_slice_mbs raises and leaves the slicing as it was."""
    w, h = 320, 192
    f = synth.desktop(w, h, 0)
    enc, ref = oracle.RefEncoder(w, h), oracle.RefEncoder(w, h)
    enc.set_idr_slice_mbs(7); ref.set_idr_slice_mbs(7)
    with pytest.raises(ValueError):
        enc.set_idr_slice_mbs(-1)
    assert enc.encode_bgra(f, True, qp=28) == ref.encode_bgra(f, True, qp=28)


def test_cropped_sizes():
    run(130, 70, [synth.gradient(130, 70, t) for t in range(3)], 24)     # coded 144x80, crop both ways
    run(16, 16, [synth.noise(16, 16, 4), synth.noise(16, 16, 5)], 20)     # one macroblock


def test_extremes_and_static():
    w, h = 64, 64
    black = np.zeros((h, w, 4), np.uint8)
    white = np.full((h, w, 4), 255, np.uint8)
    aus, _ = run(w, h, [black, black, white, white], 26)
    assert len(aus[1]) < 200          # static frame: all skipped


def test_idr_on_demand_and_structure():
    frames = [synth.desktop(128, 64, t) for t in range(5)]
    aus, _ = run(128, 64, frames, 30, idr_at=(0, 3))
    for i, au in enumerate(aus):
        types = [n[0] & 31 for n in split_nals(au)]
        if i in (0, 3):
            assert types[:2] == [7, 8] and set(types[2:]) == {5}        # SPS, PPS, IDR slices (rtc.py:394-401)
        else:
            assert set(types) == {1}
        assert au[:4] == b"\x00\x00\x00\x01"
        assert len(types) - (2 if i in (0, 3) else 0) == 4              # one slice per macroblock row
    sps = split_nals(aus[0])[0]
    assert sps[1] == 66 and sps[2] & 0xC0 == 0xC0                        # Constrained Baseline (h264.py:303-314)


def test_motion_is_found():
    """A pure translation inside the search range must cost almost nothing."""
    base = synth.noise(256, 128, 9)
    frames = [np.roll(base, (3 * t, 5 * t), axis=(0, 1)) for t in range(3)]
    aus, dec = run(256, 128, frames, 28)
    assert len(aus[1]) < len(aus[0]) // 3


@pytest.mark.parametrize("w,h,qp", [(320, 192, 30), (130, 70, 22), (208, 144, 44)])
def test_motion_search_exits_decode(w, h, qp):
    """Every exit of the P-picture motion search (zero-motion, zero-vector / temporal / anchor candidates, reduced search on new
    content, exhaustive search) on sizes whose 4x4 macroblock groups are clamped at the right / bottom edge."""
    aus, _ = run(w, h, synth.predictor_paths(w, h), qp)
    assert len(aus[1]) < 200 and len(aus[10]) < len(aus[9]) // 10          # a still costs next to nothing


def test_anchor_predictor_saves_nothing_but_time(monkeypatch):
    """The anchor / zero-vector candidates and the reduced search are shortcuts: against the same encoder with all three switched
    off (every non-static macroblock searched exhaustively) the stream may differ, but not by more than a few percent of bits."""
    w, h, qp = 320, 192, 30
    frames = synth.predictor_paths(w, h)
    fast = sum(len(a) for a in run(w, h, frames, qp)[0][1:])
    for k in ("B2V_REF_NO_ANCHOR", "B2V_REF_NO_NEWCONTENT", "B2V_REF_NO_ZCAND"):
        monkeypatch.setenv(k, "1")
    slow = sum(len(a) for a in run(w, h, frames, qp)[0][1:])
    assert abs(fast - slow) <= 0.03 * slow


def test_psnr_reasonable():
    f = synth.desktop(320, 192, 0)
    aus, dec = run(320, 192, [f], 24)
    sy, _ = oracle.csc_nv12(f)
    assert avdec.psnr(dec[0][0], sy) > 38.0


def test_cbr_rate_control_converges():
    w, h, fps, kbps = 320, 192, 30, 600
    enc = oracle.RefEncoder(w, h)
    target = kbps * 1000 // fps
    sizes = []
    for t in range(40):
        au = enc.encode_bgra(synth.desktop(w, h, t), t == 0, rc_mode=0, target_bits=target)
        sizes.append(len(au) * 8)
    avg = sum(sizes[10:]) / len(sizes[10:])
    assert 0.5 * target < avg < 1.6 * target


def test_long_run_frame_num_wraps():
    """frame_num is 8 bits (log2_max_frame_num_minus4 = 4): 600 pictures with an IDR in the middle still decode exactly."""
    w, h = 64, 48
    frames = [synth.desktop(w, h, t % 32) if t % 7 else synth.noise(w, h, t) for t in range(600)]
    run(w, h, frames, 30, idr_at=(0, 300))
