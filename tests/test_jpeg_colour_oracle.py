"""Pins the 4:2:0 colour files of oracle/jpeg_ref.c (what every stripe of the JPEG mode is) to libjpeg-turbo byte for byte: the
chroma quantiser table, the chroma DC / AC Huffman tables, the Y-Y-Y-Y-Cb-Cr interleave, the per-component DC predictors, the
3-component SOF / DHT / SOS framing and the edge padding of sizes that are not a multiple of 16.  The pictures are the ones on
which the two colour converters agree exactly (tests/jpeg_libjpeg.py): greys, and 2x2-uniform mosaics of agreeing colours."""
import numpy as np
import pytest

import oracle

cv2 = pytest.importorskip("cv2")
from tests import jpeg_libjpeg as J  # noqa: E402  (needs cv2)


@pytest.fixture(scope="module")
def palette():
    p = J.agreeing_palette(np.random.default_rng(11), 2000)
    assert len(p) > 1800              # (1961 of 2000 with libjpeg-turbo 3.x): the rule keeps almost every colour
    return p


def content(kind, w, h, request, seed=1):
    """(the palette fixture only for palette content, so that a mistake that breaks the palette leaves the grey tests apart)"""
    if kind == "grey noise":
        return J.grey_noise(w, h, seed)
    if kind == "grey desktop":
        return J.grey_desktop(w, h, seed)
    return J.mosaic(request.getfixturevalue("palette"), w, h, seed)


def check(f, quality):
    h, w = f.shape[:2]
    mine, ref = oracle.jpeg_encode_bgra(f, quality), J.padded_reference(f, w, h, quality)
    assert mine == ref, f"{w}x{h} quality {quality}: {J.difference(mine, ref, w)}"


@pytest.mark.parametrize("kind", ["grey noise", "grey desktop", "palette"])
@pytest.mark.parametrize("quality", range(1, 101))
def test_every_quality(kind, quality, request):
    """Every quantiser table of both kinds, including the clamps to 255 (luma below quality 24, chroma below 20) and to 1."""
    check(content(kind, 64, 48, request), quality)


@pytest.mark.parametrize("w,h", [(16, 16), (130, 70), (642, 362), (1920, 1080), (7680, 64)])
@pytest.mark.parametrize("quality", [1, 24, 50, 51, 100])
@pytest.mark.parametrize("kind", ["grey noise", "palette"])
def test_sizes(kind, w, h, quality, request):
    """130x70, 642x362 and 1920x1080 end in partial MCUs (edge padding); 7680x64 is 480 MCUs wide."""
    check(content(kind, w, h, request, seed=w + h), quality)


def test_largest_dc_differences_in_both_dc_tables():
    """Category-11 DC differences at quality 100: an 8x8 black / white checkerboard in luma, and 16x16 red / blue alternation,
    whose Cb and Cr swing between their extremes from one MCU to the next."""
    yy, xx = np.indices((64, 128))
    check(J.grey(((yy // 8 + xx // 8) % 2 * 255).astype(np.uint8)), 100)
    red, blue = np.array([0, 0, 255], np.uint8), np.array([255, 0, 0], np.uint8)
    for c in (red, blue):               # both convert identically in both coders, so the rule would keep them
        f = J.bgra(np.broadcast_to(c, (16, 16, 3)))
        assert oracle.jpeg_encode_bgra(f, 100) == J.libjpeg_420(f, 100)
    alt = ((yy // 16 + xx // 16) % 2).astype(bool)
    check(J.bgra(np.where(alt[..., None], red, blue)), 100)


def test_binary_grey_noise_at_quality_100():
    """The densest content found: about 81 bytes per block, the most any delivered stripe carries."""
    f = J.grey_noise(256, 128, 5, binary=True)
    check(f, 100)
    assert len(oracle.jpeg_encode_bgra(f, 100)) / (256 * 128 * 6 // 256) > 70
