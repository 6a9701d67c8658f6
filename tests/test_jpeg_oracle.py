"""Pins oracle/jpeg_ref.c (the JPEG stripe mode, CaptureSettings.output_mode = 0): the single-component output must be
byte-identical to libjpeg-turbo's (cv2.imencode) for the same grey image and quality — same integer DCT, quantisation rule,
Annex K tables, Huffman coding, stuffing and JFIF framing; 4:2:0 streams must decode (libjpeg-turbo) close to the source."""
import numpy as np
import pytest

import oracle
from tests import synth

cv2 = pytest.importorskip("cv2")


def grey_plane(w, h, seed):
    f = synth.desktop(w, h, seed) if w >= 128 else synth.noise(w, h, seed)
    cw, ch = (w + 15) & ~15, (h + 15) & ~15
    return np.ascontiguousarray(oracle.csc_nv12(f, coded_w=cw, coded_h=ch, matrix=1)[0])


@pytest.mark.parametrize("w,h", [(16, 16), (64, 48), (130, 78), (320, 192), (642, 362)])
@pytest.mark.parametrize("quality", [5, 30, 60, 90, 100])
def test_grey_jpeg_is_byte_identical_to_libjpeg_turbo(w, h, quality):
    g = grey_plane(w, h, 3)
    mine = oracle.jpeg_encode(g, None, w, h, quality)
    ok, ref = cv2.imencode(".jpg", g[:h, :w], [cv2.IMWRITE_JPEG_QUALITY, quality])
    assert ok and mine == ref.tobytes()


def test_noise_and_extremes_byte_identical():
    rng = np.random.default_rng(7)
    for img in (rng.integers(0, 256, (96, 160), dtype=np.uint8), np.zeros((32, 32), np.uint8), np.full((32, 32), 255, np.uint8),
                np.tile(np.array([[0, 255], [255, 0]], np.uint8), (24, 40))):        # the checkerboard drives the largest AC magnitudes
        h, w = img.shape
        for q in (50, 100):
            ok, ref = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])
            assert oracle.jpeg_encode(img, None, w, h, q) == ref.tobytes()


@pytest.mark.parametrize("w,h", [(64, 48), (320, 192), (130, 70)])
@pytest.mark.parametrize("quality", [60, 90])
def test_colour_420_decodes_as_well_as_libjpeg_turbos_own(w, h, quality):
    f = synth.gradient(w, h, 2)
    f[h // 4: h // 2, w // 4: w // 2] = synth.bars(w, h, 1)[h // 4: h // 2, w // 4: w // 2]
    data = oracle.jpeg_encode_bgra(f, quality)
    assert data[:2] == b"\xff\xd8" and data[-2:] == b"\xff\xd9"

    def psnr(jpg):
        dec = cv2.imdecode(np.frombuffer(jpg, np.uint8), cv2.IMREAD_COLOR)
        assert dec is not None and dec.shape == (h, w, 3)
        return 10 * np.log10(255 ** 2 / max(np.mean((dec.astype(float) - f[..., :3].astype(float)) ** 2), 1e-9))
    # the same picture through libjpeg-turbo's own colour path (4:2:0, same quality): this coder must decode as close to the
    # source (within half a dB: different chroma rounding, same DCT / tables) at a comparable size
    ok, ref = cv2.imencode(".jpg", f[..., :3], [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])
    assert psnr(data) > psnr(ref.tobytes()) - 0.5
    assert abs(len(data) - len(ref)) <= 0.12 * len(ref) + 64


def test_jfif_matrix_known_answers():
    """JFIF full-range BT.601: white (255,128,128), black (0,128,128), red (76,85,255), green (150,44,21), blue (29,255,107)."""
    for bgr, want in (((255, 255, 255), (255, 128, 128)), ((0, 0, 0), (0, 128, 128)), ((0, 0, 255), (76, 85, 255)), ((0, 255, 0), (150, 44, 21)), ((255, 0, 0), (29, 255, 107))):
        f = np.zeros((16, 16, 4), np.uint8)
        f[..., :3] = bgr
        y, uv = oracle.csc_nv12(f, matrix=1)
        assert (int(y[0, 0]), int(uv[0, 0]), int(uv[0, 1])) == want


def test_jfif_matrix_within_one_lsb_of_float64():
    """Matrix 1 against a float64 evaluation of JFIF full-range BT.601 with 2x2 box chroma (the mean of the four pixels'
    Cb / Cr): never more than 1 LSB off, and the correctly rounded value almost everywhere."""
    f = synth.noise(256, 128, 3)
    y, uv = oracle.csc_nv12(f, matrix=1)
    b, g, r = [f[..., i].astype(np.float64) for i in range(3)]
    fy = 0.299 * r + 0.587 * g + 0.114 * b
    box = lambda a: (a[0::2, 0::2] + a[0::2, 1::2] + a[1::2, 0::2] + a[1::2, 1::2]) / 4
    fcb, fcr = box(128 + (b - fy) / 1.772), box(128 + (r - fy) / 1.402)
    for got, want in ((y, fy), (uv[:, 0::2], fcb), (uv[:, 1::2], fcr)):
        assert np.abs(got - want).max() <= 1.0
        assert (got != np.rint(want)).mean() < 0.01


def test_jfif_matrix_keeps_every_grey():
    """Y = v and Cb = Cr = 128 for every grey level: the identity on which the grey comparisons with libjpeg-turbo rest."""
    f = np.zeros((2, 512, 4), np.uint8)
    f[..., :3] = (np.arange(512) // 2).astype(np.uint8)[None, :, None]
    y, uv = oracle.csc_nv12(f, matrix=1)
    assert (y == f[..., 0]).all() and (uv == 128).all()
