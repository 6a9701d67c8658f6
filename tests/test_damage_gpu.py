"""GPU: damage rectangles (B2V_FLAG_DAMAGE).  A damage submit whose rectangles cover every changed pixel codes exactly what a
whole-frame submit codes: against the unchanged oracle through tests/damage_scenario.py (slots poisoned outside the
rectangles), and GPU against GPU for the modes the oracle driver does not cover.  Then the rules: B2V_ESTATE, h2d_bytes,
kernel_launches, and ScreenCapture with a DamageFrameSource."""
import numpy as np
import pytest

from selkies_b200 import _native as N
from selkies_b200.session import Session, normalize_rects
from tests import damage_scenario as D
from tests import scenario as S
from tests import synth

pytestmark = pytest.mark.gpu


# ---- 1. parity with the oracle --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [
    S.Config(256, 160, qp=28),
    S.Config(16, 16, qp=24),
    S.Config(250, 142, qp=26),                                            # cropped: coded 256 x 144
    S.Config(320, 192, dst_width=224, dst_height=128, qp=28),            # down-scaled
    S.Config(160, 96, dst_width=272, dst_height=176, qp=30),             # up-scaled
    S.Config(256, 192, qp=28, stripe_rows=4, header_mode=S.HDR_PIXELFLUX),
], ids=["cqp", "16x16", "cropped", "down", "up", "striped"])
def test_parity_with_the_oracle(cfg):
    D.run(cfg, S.stream(D.desktop_session(cfg.width, cfg.height)))


def test_cbr_idr_request_and_gop():
    f = D.desktop_session(320, 176)
    ev = S.stream(f[:5]) + [S.request_idr()] + S.stream(f[5:8]) + [S.set_gop(3)] + S.stream(f[8:])
    D.run(S.Config(320, 176, rc_mode=S.CBR, kbps=3000), ev)


def test_paint_over_on_a_static_stretch():
    f = D.desktop_session(256, 144)
    D.run(S.Config(256, 144, paint=(2, 18, 2)), S.stream(f[:4] + [f[3]] * 5 + f[4:6]))


def test_resize_mid_stream():
    a, b = D.desktop_session(256, 144), D.desktop_session(320, 176, seed=1)
    D.run(S.Config(256, 144, qp=27), S.stream(a[:6]) + [S.resize(320, 176)] + S.stream(b[:6]) + [S.resize(256, 144, 192, 112)] +
          S.stream(a[6:]))


def test_headline_4k():
    D.run(S.Config(3840, 2160, rc_mode=S.CBR, kbps=20000), S.stream(D.desktop_session(3840, 2160)[:8]), decode=False)


# ---- 2. whole against damage, GPU against GPU -------------------------------------------------------------------------------------
def _pair(frames, submit_whole, submit_damage, **kw):
    """The deliveries of two sessions with the same settings: one fed whole pictures, one damage submits."""
    out = []
    for damage_flag, submit in ((False, submit_whole), (True, submit_damage)):
        with Session(frames[0].shape[1], frames[0].shape[0], damage=damage_flag, **kw) as s:
            prev = None
            for f in frames:
                submit(s, f, None if prev is None else D.damage(prev, f))
                prev = f
            s.flush()
            st = s.stats()
            out.append(([(r.data, r.is_key, r.qp, r.y_start, r.height, r.quality) for r in s.take_frames()],
                        st["kernel_launches"], st["frames_delivered"]))
    return out


def _ring_whole(s, f, rects):
    s.submit(f)


def _ring_damage(s, f, rects, rng=np.random.default_rng(3)):
    D.submit_poisoned(s, f, rects, rng)


@pytest.mark.parametrize("kw", [
    dict(flags=N.B2V_FLAG_JPEG, stripe_rows=3, crf=70, header_mode=N.B2V_HDR_PIXELFLUX),
    dict(droppable=True, rc_mode=N.B2V_RC_CQP, crf=27),
    dict(wide_motion=True, rc_mode=N.B2V_RC_CQP, crf=28),
    dict(long_term_ref=True, rc_mode=N.B2V_RC_CQP, crf=26),
    dict(quality=True, rc_mode=N.B2V_RC_CBR, bitrate_kbps=4000),
    dict(dst_width=192, dst_height=112, quality=True, rc_mode=N.B2V_RC_CQP, crf=30),
], ids=["jpeg", "droppable", "wide_motion", "long_term_ref", "quality", "quality_scaled"])
def test_ring_whole_equals_damage(kw):
    frames = D.desktop_session(320, 192)
    whole, dmg = _pair(frames, _ring_whole, _ring_damage, **kw)
    assert len(whole[0]) > 0 and whole == dmg


def test_no_encode_whole_equals_damage():
    # NV12 pictures have no readback of their own: compare what the session reports, and the stream of a coded session fed
    # the same way (test_ring_whole_equals_damage) shows the pictures themselves are equal
    frames = D.desktop_session(256, 144)
    whole, dmg = _pair(frames, _ring_whole, _ring_damage, flags=N.B2V_FLAG_NO_ENCODE)
    assert whole == dmg and whole[2] == len(frames) and whole[1] == len(frames)


@pytest.mark.parametrize("fmt", ["BGRA", "RGBA", "BGR", "RGB"])
def test_device_whole_equals_damage(fmt):
    from tests.device_scenario import device_surface
    frames = D.desktop_session(250, 142)
    margin = (3, 5)
    surf = {id(f): device_surface(f, fmt, margin) for f in frames}

    def sub(s, f, rects):
        s.submit_device(surf[id(f)], pixel_format=fmt, origin=margin, damage=rects)
    whole, dmg = _pair(frames, lambda s, f, r: sub(s, f, None), sub, rc_mode=N.B2V_RC_CQP, crf=27)
    assert len(whole[0]) == len(frames) and whole == dmg


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_tensor_whole_equals_damage(dtype):
    from tests.tensor_scenario import device_tensor, host_tensor
    frames = D.desktop_session(256, 144)
    tens, quant = {}, []
    for f in frames:                     # the quantised frames decide the damage; the tensors are what is submitted
        if id(f) not in tens:
            t, q = host_tensor(f, dtype, "RGB")
            tens[id(f)] = (device_tensor(t, "CHW", (2, 1))[0], q)
        quant.append(tens[id(f)][1])
    by_q = {id(q): tens[id(f)][0] for f, q in zip(frames, quant)}

    def sub(s, q, rects):
        s.submit_tensor(by_q[id(q)], channels="RGB", layout="CHW", origin=(2, 1), damage=rects)
    whole, dmg = _pair(quant, lambda s, q, r: sub(s, q, None), sub, rc_mode=N.B2V_RC_CQP, crf=28)
    assert len(whole[0]) == len(frames) and whole == dmg


# ---- 3. the rules -----------------------------------------------------------------------------------------------------------------
def test_a_ring_damage_submit_needs_a_ring_picture_before_it():
    w, h = 64, 48
    f = synth.desktop(w, h, 0)
    with Session(w, h, damage=True, rc_mode=N.B2V_RC_CQP) as s:
        def refused():
            slot, view = s.acquire()
            with pytest.raises(N.B2VError) as e:
                s.submit_slot(slot, damage=[(0, 0, 8, 8)])
            assert e.value.code == N.B2V_ESTATE
            view[...] = f                  # the slot is still held: fill it whole and submit it again
            s.submit_slot(slot)
        refused()                          # after create
        s.submit(f, damage=[(1, 1, 4, 4)])
        s.set_resolution(96, 64)
        f = synth.desktop(96, 64, 0)
        refused()                          # after a resize
        import torch
        s.submit_device(torch.from_numpy(f).cuda())
        refused()                          # after a device picture
        s.submit(f, damage=[])
        s.flush()
        assert len(s.take_frames()) == 6
    with Session(w, h, rc_mode=N.B2V_RC_CQP) as s:                 # no flag
        slot, _ = s.acquire()
        with pytest.raises(N.B2VError) as e:
            s.submit_slot(slot, damage=[(0, 0, 8, 8)])
        assert e.value.code == N.B2V_EINVAL and "B2V_FLAG_DAMAGE" in str(e.value)
        s.release_slot(slot)


def test_h2d_bytes_and_kernel_launches():
    w, h = 320, 192
    frames = D.desktop_session(w, h)
    launches = {}
    for flag in (False, True):
        with Session(w, h, damage=flag, rc_mode=N.B2V_RC_CQP) as s:
            prev, per = None, []
            for f in frames:
                before = s.stats()
                rects = None if prev is None or not flag else D.damage(prev, f)
                D.submit_poisoned(s, f, rects, np.random.default_rng(0))
                s.flush()
                after = s.stats()
                copied = after["h2d_bytes"] - before["h2d_bytes"]
                if rects is None:
                    assert copied == w * h * 4
                else:                        # what submit_poisoned submitted: clipped, merged past the cap
                    assert copied == 4 * sum(rw * rh for _, _, rw, rh in normalize_rects(rects, w, h))
                per.append(after["kernel_launches"] - before["kernel_launches"])
                prev = f
            launches[flag] = per
    assert launches[True] == launches[False]


def test_screen_capture_with_a_damage_source_across_a_resize():
    from selkies_b200.pixelflux_compat import CaptureSettings, DamageFrameSource, FrameSource, ScreenCapture
    sizes = {(256, 144): D.desktop_session(256, 144), (320, 176): D.desktop_session(320, 176, seed=2)}
    n = len(sizes[(256, 144)])

    class Whole(FrameSource):
        live = False                       # the capture thread's first call ends its loop: the test drives the pictures

        def fill(self, view, index):
            if self.live:
                view[...] = sizes[(self.width, self.height)][index % n]
            return self.live

    class Damage(DamageFrameSource):
        live, rng = False, np.random.default_rng(4)

        def fill_damage(self, view, index, whole):
            if not self.live:
                return None
            fr = sizes[(self.width, self.height)]
            f = fr[index % n]
            view[...] = self.rng.integers(0, 256, view.shape, dtype=np.uint8)
            if whole:
                view[...] = f
                return []
            rects = D.damage(fr[(index - 1) % n], f)
            for x, y, w, h in rects:
                view[y:y + h, x:x + w] = f[y:y + h, x:x + w]
            return rects

    def run(src):
        got = []
        cs = ScreenCapture(src)
        st = CaptureSettings()
        st.capture_width, st.capture_height, st.h264_crf = 256, 144, 27
        cs.start_capture(st, lambda r, _u: got.append(bytes(r.contents.data[:r.contents.size])))
        cs._thread.join()
        src.live = True
        for i in range(n):
            assert cs._encode_next(cs._session, i)
        cs.update_resolution(320, 176)
        for i in range(n):
            assert cs._encode_next(cs._session, i)
        cs.stop_capture()
        return got
    a, b = run(Whole()), run(Damage())
    assert len(a) == 2 * n and a == b
