"""GPU parity: the CUDA H.264 encoder vs oracle/h264_ref.c — access units, QP, key flags and reconstruction bit-exact, through
the C-ABI (ring ingest -> fused CSC -> encode -> callback), driven by tests/scenario.py."""
import numpy as np
import pytest

import oracle
from oracle import avdec
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import scenario as S
from tests import synth

pytestmark = pytest.mark.gpu


def encode(w, h, frames, idr_at=(), **cfg):
    """Both encoders over `frames` (an IDR requested before every picture in idr_at); returns the oracle's Expected records."""
    return S.pictures(S.run(S.Config(w, h, **cfg), S.stream(frames, idr_at)))


@pytest.mark.parametrize("w,h", [(16, 16), (64, 48), (130, 70), (320, 192)])
@pytest.mark.parametrize("qp", [12, 28, 44])
def test_intra_bit_exact(w, h, qp):
    frames = [synth.noise(w, h, 3), synth.desktop(w, h, 1)]
    xs = encode(w, h, frames, idr_at=(1,), qp=qp, slice_rows=1)
    assert all(x.is_key for x in xs)


@pytest.mark.parametrize("w,h,slice_rows", [(64, 48, 1), (160, 96, 1), (160, 96, 2), (320, 192, 3), (130, 70, 100), (64, 48, 0), (320, 192, 0), (640, 368, 0), (1280, 720, 0)])
def test_p_frames_bit_exact(w, h, slice_rows):
    frames = [synth.desktop(w, h, t) for t in range(5)]
    xs = encode(w, h, frames, qp=30, slice_rows=slice_rows)
    assert [x.is_key for x in xs] == [True, False, False, False, False]


def test_escape_boundaries_bit_exact():
    """Emulation-prevention bytes where the byte-stream copy splits its work: zero runs that start in the previous thread's
    16-byte chunk, and escapes in the second 4096-byte round of a slice (test_escape_cases_oracle.py checks that this
    content reaches both)."""
    w, h = 1280, 720
    xs = encode(w, h, [synth.desktop(w, h, t) for t in range(3)], qp=10)
    assert [x.is_key for x in xs] == [True, False, False]


def test_motion_and_noise_bit_exact():
    base = synth.noise(256, 128, 9)
    encode(256, 128, [np.roll(base, (3 * t, -5 * t), axis=(0, 1)) for t in range(4)], qp=26, slice_rows=1)
    encode(192, 112, [synth.bars(192, 112, t) for t in range(6)], qp=22, slice_rows=2)


@pytest.mark.parametrize("w,h,qp,slice_rows", [(320, 192, 30, 1), (130, 70, 22, 1), (208, 144, 44, 2), (640, 368, 36, 1)])
def test_motion_search_exits_bit_exact(w, h, qp, slice_rows):
    """Every exit of k_inter_mb's motion search — zero-motion, zero-vector / temporal / anchor candidates, the reduced search on new
    content, the exhaustive search — incl. sizes whose 4x4 macroblock groups are clamped at the right / bottom edge (synth.predictor_paths)."""
    encode(w, h, synth.predictor_paths(w, h), qp=qp, slice_rows=slice_rows)


@pytest.mark.parametrize("qp,slice_rows", [(0, 1), (6, 2), (14, 1)])
def test_pcm_fallback_bit_exact(qp, slice_rows):
    """Macroblocks whose CAVLC size bound exceeds 3200 bits are sent as I_PCM (I and P slices)."""
    w, h = 128, 96
    frames = []
    for t in range(3):
        f = synth.desktop(w, h, t)
        f[:48] = synth.noise(w, 48, t + 5)          # top half: incompressible at low QP -> I_PCM; bottom: ordinary
        frames.append(f)
    xs = encode(w, h, frames, qp=qp, slice_rows=slice_rows)
    if qp <= 6:
        assert len(xs[1].au) > 24 * 384              # the P picture still carries the raw macroblocks


def natural_frames(w, h):
    """Anti-aliased text and a photo-like texture: content where Intra4x4 wins the rate-distortion decision."""
    cv2 = pytest.importorskip("cv2")
    img = np.full((h, w, 3), 245, np.uint8)
    for i, y in enumerate(range(20, h, 20)):
        cv2.putText(img, "The quick brown fox jumps over the lazy dog 0123456789"[i % 9:], (6, y), cv2.FONT_HERSHEY_SIMPLEX, 0.5, (20, 20, 20), 1, cv2.LINE_AA)
    cv2.circle(img, (w * 3 // 4, h // 2), h // 5, (200, 80, 40), -1, cv2.LINE_AA)
    text = np.dstack([img, np.full((h, w), 255, np.uint8)])
    rng = np.random.default_rng(3)
    a = cv2.GaussianBlur(rng.normal(0, 1, (h, w, 3)).astype(np.float32), (0, 0), 5) * 800 + \
        cv2.GaussianBlur(rng.normal(0, 1, (h, w, 3)).astype(np.float32), (0, 0), 1.2) * 40 + 128
    photo = np.dstack([np.clip(a, 0, 255).astype(np.uint8), np.full((h, w), 255, np.uint8)])
    return [text, photo]


@pytest.mark.parametrize("slice_rows", [1, 3, 100])
@pytest.mark.parametrize("qp", [20, 34])
def test_intra4x4_bit_exact(slice_rows, qp):
    """Intra4x4 (9 modes, above-right availability across macroblock and slice boundaries) + the I4/I16 RD decision."""
    w, h = 320, 192
    encode(w, h, natural_frames(w, h) + [synth.gradient(w, h, 1)], idr_at=(1, 2), qp=qp, slice_rows=slice_rows)


def test_subpel_motion_bit_exact():
    """A pan by (1.37, 0.61) samples per picture: the quarter-sample refinement (6-tap interpolation) must be taken and must
    match the oracle; the P pictures cost a fraction of what integer-only vectors would need."""
    cv2 = pytest.importorskip("cv2")
    w, h = 320, 192
    rng = np.random.default_rng(5)
    big = cv2.GaussianBlur(rng.normal(0, 1, (h + 96, w + 96, 3)).astype(np.float32), (0, 0), 5) * 900 + \
        cv2.GaussianBlur(rng.normal(0, 1, (h + 96, w + 96, 3)).astype(np.float32), (0, 0), 1.2) * 40 + 128
    frames = []
    for t in range(5):
        a = cv2.warpAffine(big, np.float32([[1, 0, -(24 + 1.37 * t)], [0, 1, -(24 + 0.61 * t)]]), (w, h), flags=cv2.INTER_CUBIC)
        frames.append(np.dstack([np.clip(a, 0, 255).astype(np.uint8), np.full((h, w), 255, np.uint8)]))
    xs = encode(w, h, frames, qp=26, slice_rows=2)
    assert sum(len(x.au) for x in xs[1:]) < len(xs[0].au) // 2          # 4 P pictures together under half an IDR


def test_static_scene_is_skipped():
    f = synth.desktop(320, 192, 0)
    xs = encode(320, 192, [f, f, f], qp=30, slice_rows=1)
    assert len(xs[2].au) < 150


def test_cbr_rate_control_bit_exact():
    w, h = 320, 192
    frames = [synth.desktop(w, h, t) for t in range(12)]
    xs = encode(w, h, frames, rc_mode=S.CBR, kbps=600, fps=30.0, slice_rows=1)
    assert len({x.qp for x in xs}) > 1           # the controller actually moved


def test_cbr_midstream_idr_is_bounded_and_bit_exact():
    """A key frame requested in mid-stream (PLI -> dynamic_idr_frame, rtc.py:601-603) is coded no finer than a fresh start
    with 4x the picture budget; the controller then resumes from its running QP."""
    w, h = 320, 192
    frames = [synth.gradient(w, h, t) for t in range(14)]
    xs = encode(w, h, frames, idr_at=(9,), rc_mode=S.CBR, kbps=3000, fps=30.0, slice_rows=1)
    assert xs[9].is_key and xs[9].qp >= xs[8].qp and xs[10].qp <= xs[9].qp


def test_gpu_stream_decodes_to_its_reconstruction():
    w, h = 320, 184                               # cropped height
    frames = [synth.desktop(w, h, t) for t in range(4)]
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=27) as s:
        recs = []
        for f in frames:
            s.submit(f)
            s.flush()
            recs.append(s.recon())
        got = s.take_frames()
    dec = avdec.decode_stream([g.data for g in got], quiet=True)
    assert len(dec) == len(frames)
    for (Y, U, V), (ry, ruv) in zip(dec, recs):
        assert np.array_equal(Y, ry[:h, :w]) and np.array_equal(U, ruv[: h // 2, 0:w:2]) and np.array_equal(V, ruv[: h // 2, 1:w:2])
    sy, _ = oracle.csc_nv12(frames[-1])
    assert avdec.psnr(dec[-1][0], sy) > 33.0


def test_1080p_one_idr_one_p_bit_exact():
    """BASELINE config 1 size (coded 1920x1088, bottom crop 8)."""
    w, h = 1920, 1080
    encode(w, h, [synth.desktop(w, h, 0), synth.desktop(w, h, 1)], qp=30, slice_rows=1)


def test_pixelflux_header_mode():
    """Each access unit behind the 10-byte header 04 | is_key | frame_id | y_start 0 | width | height (checked by the driver)."""
    w, h = 64, 48
    xs = encode(w, h, [synth.noise(w, h, 1), synth.noise(w, h, 2)], qp=30, header_mode=S.HDR_PIXELFLUX)
    assert [x.is_key for x in xs] == [True, False]


def test_8k_encode_decodes_to_its_reconstruction():
    """Maximum size the reference allows (7680x4320, selkies.py:281; level 6.2): property check instead of a full oracle run —
    the stream decodes and the decoder output equals the encoder's reconstruction."""
    w, h = 7680, 4320
    tile = synth.desktop(1920, 1080, 0)
    f0 = np.tile(tile, (4, 4, 1))
    f1 = np.roll(f0, (6, -10), axis=(0, 1))
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=36) as s:
        recs = []
        for f in (f0, f1):
            s.submit(f)
            s.flush()
            recs.append(s.recon())
        got = s.take_frames()
    assert got[0].is_key and not got[1].is_key
    dec = avdec.decode_stream([g.data for g in got], quiet=True)
    assert len(dec) == 2
    for (Y, U, V), (ry, ruv) in zip(dec, recs):
        assert np.array_equal(Y, ry[:h, :w]) and np.array_equal(U, ruv[: h // 2, 0:w:2]) and np.array_equal(V, ruv[: h // 2, 1:w:2])
    assert len(got[1].data) < len(got[0].data) // 3          # the translation was found


def test_paintover_bit_exact():
    """CQP paint-over (CaptureSettings.use_paint_over_quality, selkies.py:3226-3229): after `trigger` all-skipped pictures one
    picture is coded at the paint-over QP, once, until the scene moves again."""
    w, h = 320, 192
    a, b = natural_frames(w, h)[0], synth.desktop(w, h, 2)
    xs = encode(w, h, [a] * 7 + [b] * 11, qp=32, slice_rows=1, paint=(3, 16, 1))
    qps = [x.qp for x in xs]
    painted = [i for i, q in enumerate(qps) if q == 16]
    assert len(painted) == 2 and painted[0] in (4, 5) and painted[1] >= 10 and painted[1] < 17 and set(qps) == {16, 32}
    k = painted[0]
    dec = avdec.decode_stream([x.au for x in xs], quiet=True)
    sy, _ = oracle.csc_nv12(a)
    assert avdec.psnr(dec[k][0], sy) > avdec.psnr(dec[k - 1][0], sy) + 4.0  # the static text got sharper
    assert len(xs[k + 1].au) < 150                                           # and is skipped again afterwards


def test_paintover_burst_bit_exact():
    """h264_paintover_burst_frames (selkies.py:3217): `burst` consecutive pictures at the paint-over QP once the trigger is
    reached; motion cancels what is left of a burst.  Also in CBR mode, where the paint-over QP applies when it is finer."""
    w, h = 320, 192
    a = natural_frames(w, h)[0]
    frames = [a] * 10 + [synth.desktop(w, h, t) for t in range(6)] + [a] * 22      # static, six pictures of motion, static again
    for rc_mode in (S.CQP, S.CBR):
        xs = encode(w, h, frames, rc_mode=rc_mode, qp=34, kbps=300, fps=30.0, slice_rows=1, paint=(3, 20, 3))
        qps = [x.qp for x in xs]
        if rc_mode == S.CQP:
            assert qps[5:8] == [20, 20, 20] and qps[8] == 34 and qps[4] == 34, qps       # trigger after pictures 1..3, two pictures of feedback delay
            # motion never paints; the second static period paints again once its last small refinements have died out
            assert qps[8:22] == [34] * 14 and qps[22:].count(20) == 3, qps
            k = qps.index(20, 22)
            assert qps[k:k + 3] == [20, 20, 20], qps                                      # ... as one burst
        else:
            assert min(qps[5:8]) == 20, qps


@pytest.mark.parametrize("w,h,mbs,slice_rows", [(320, 192, 7, 0), (320, 192, 10, 1), (130, 70, 3, 0), (640, 368, 40, 3), (320, 192, 0, 2)])
def test_idr_subrow_slices_bit_exact(w, h, mbs, slice_rows):
    """IDR pictures cut into slices shorter than a macroblock row (b2v_settings.idr_slice_mbs): left/top availability, nC
    contexts, Intra4x4 mode prediction and first_mb_in_slice all follow the finer slice grid; P pictures keep `slice_rows` whole rows
    (0 = the default rule: 8)."""
    frames = natural_frames(w, h)[:1] + [synth.desktop(w, h, 1), synth.desktop(w, h, 2), synth.noise(w, h, 7)]
    xs = encode(w, h, frames, idr_at=(3,), qp=27, slice_rows=slice_rows, idr_slice_mbs=mbs)
    if mbs > 0:
        au = xs[0].au
        n_idr_slices = sum(1 for i in range(len(au) - 4) if au[i:i + 3] == b"\x00\x00\x01" and (au[i + 3] & 31) == 5)
        assert n_idr_slices == ((h + 15) // 16) * -(-((w + 15) // 16) // mbs)


def test_idr_subrow_slices_striped_bit_exact():
    """Default slicing (one slice per stripe in P pictures) with IDR slices of 6 macroblocks."""
    w, h = 320, 192
    encode(w, h, [synth.desktop(w, h, t) for t in range(3)], qp=30, idr_slice_mbs=6, stripe_rows=4)


@pytest.mark.parametrize("name,kbps", [("desktop_scroll", 8000), ("gradient_pan", 8000), ("gradient_pan", 20000)])
def test_cbr_holds_its_target_1080p(name, kbps):
    """VERDICT r1 #7: CBR must be CBR.  1080p60, 180 pictures: the second half within +-10 % of the target, no one-second window after
    the first second above +20 % (knob range: settings.py:49)."""
    w, h, fps, n = 1920, 1080, 60.0, 180
    gen = synth.desktop if name == "desktop_scroll" else synth.gradient
    with Session(w, h, rc_mode=N.B2V_RC_CBR, bitrate_kbps=kbps, fps=fps, collect=True) as s:
        for t in range(n):
            s.submit(gen(w, h, t))
        s.flush()
        got = s.take_frames()
    sizes = np.array([len(g.data) for g in got], float)
    tb = kbps * 1000.0 / fps / 8.0
    steady = sizes[n // 2:].mean() / tb
    win = int(fps)
    worst = max(sizes[i:i + win].sum() / (tb * win) for i in range(win, n - win + 1))
    qps = [g.qp for g in got[n // 2:]]
    assert max(qps) < 51, qps                                # the controller is not pinned at the coarse limit on these runs
    assert steady <= 1.1 and (steady >= 0.9 or min(qps) <= 10), (steady, qps[-10:])   # under-spending only when the QP floor is reached
    assert worst <= 1.2, worst
