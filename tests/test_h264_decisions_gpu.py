"""The checks of tests/test_h264_decisions.py on the CUDA encoder's own bytes: the access units come from
`Session.take_frames()` and the reconstruction from `Session.recon()`, not from the oracle."""
import numpy as np
import pytest

from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import scenario as S
from tests import test_h264_decisions as D

pytestmark = pytest.mark.gpu


def _session(cfg: S.Config) -> Session:
    p = cfg.paint
    return Session(cfg.width, cfg.height, fps=cfg.fps, rc_mode=cfg.rc_mode, bitrate_kbps=cfg.kbps, crf=cfg.qp, gop=cfg.gop,
                   slice_rows=cfg.slice_rows, idr_slice_mbs=cfg.idr_slice_mbs, stripe_rows=cfg.stripe_rows,
                   paintover_trigger_frames=p[0], paintover_crf=p[1], paintover_burst_frames=p[2], flags=cfg.flags)


def encode_gpu(cfg: S.Config, frames, idr_at=(0,), qps=None) -> D.Encoded:
    with _session(cfg) as s:
        cw, ch = s.coded_size()
        out = D.Encoded(cfg.width, cfg.height, cw, ch)
        out.flags = cfg.flags
        for i, f in enumerate(frames):
            if i in idr_at and i > 0:
                s.flush()
                s.request_idr()
            if qps is not None:
                s.set_qp(qps[i])
            s.submit(f)
            out.sources.append(D.source_nv12(f, cw, ch))
        s.flush()
        for r in s.take_frames():
            out.add(r.frame_id, r.y_start, r.data)
        out.recon = s.recon()
    for items in out.bands.values():
        items.sort(key=lambda t: t[0])
    return out


class GpuEnc:
    """One CQP session, picture by picture (the D.OracleEnc interface)."""

    def __init__(self, w, h, qp, slice_rows=0, stripe_rows=0, wide=False):
        self.s = Session(w, h, rc_mode=N.B2V_RC_CQP, crf=qp, slice_rows=slice_rows, stripe_rows=stripe_rows, wide_motion=wide)
        self.first = True

    def encode(self, frame, idr):
        if idr and not self.first:
            self.s.request_idr()
        self.first = False
        self.s.submit(frame)
        self.s.flush()
        return {r.y_start: r.data for r in self.s.take_frames()}

    def recon(self):
        return self.s.recon()

    def close(self):
        self.s.close()


@pytest.mark.parametrize("case", D.CASES, ids=[c[0] for c in D.CASES])
def test_gpu_decisions(case):
    e, st = D.run_case(encode_gpu, case)
    D.check_recon(e, st)
    assert st.pictures >= len(case[2])
    D.assert_targets(case[0], st)


def test_gpu_motion_recovery():
    D.motion_recovery(GpuEnc)


@pytest.mark.parametrize("w,h,shifts,gate_at", [(448, 128, D.WIDE_SHIFTS_ACROSS, (13, 1)), (96, 640, D.WIDE_SHIFTS_DOWN, None)],
                         ids=["across", "down"])
def test_gpu_wide_motion_recovery(w, h, shifts, gate_at):
    D.motion_recovery(GpuEnc, w=w, h=h, wide=True, shifts=shifts, gate_at=gate_at)


@pytest.mark.parametrize("w,h,stripe_rows", [(130, 70, 0), (200, 112, 3)])
def test_gpu_search_optimality(w, h, stripe_rows):
    D.search_optimality(GpuEnc, w, h, stripe_rows)


@pytest.mark.parametrize("w,h,stripe_rows,shift,blocky", D.WIDE_OPTIMALITY)
def test_gpu_wide_search_optimality(w, h, stripe_rows, shift, blocky):
    D.search_optimality(GpuEnc, w, h, stripe_rows, wide=True, shift=shift, blocky=blocky)


@pytest.mark.parametrize("w,h,stripe_rows", [(3840, 64, 0), (3840, 2160, 8)])
def test_gpu_wide_pictures_and_bands_carry_a_level_that_holds_them(w, h, stripe_rows):
    from tests.h264_syntax import parse_sps, split_annexb, unescape
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=40, stripe_rows=stripe_rows) as s:
        s.submit(np.zeros((h, w, 4), np.uint8))
        s.flush()
        aus = [r.data for r in s.take_frames()]
    spss = [parse_sps(unescape(n)) for au in aus for n in split_annexb(au) if n[0] & 31 == 7]
    assert len(spss) == (-(-h // (16 * stripe_rows)) if stripe_rows else 1)
    for sps in spss:
        assert D.level_ok(sps.level_idc, sps.mbw, sps.mbh), (sps.level_idc, sps.mbw, sps.mbh)
        assert sps.level_idc == D.smallest_level(sps.mbw, sps.mbh)
