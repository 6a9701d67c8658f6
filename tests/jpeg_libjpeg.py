"""libjpeg-turbo (through cv2.imencode) as a direct reference for the 4:2:0 files of the JPEG stripe mode.

libjpeg-turbo converts colour per pixel and then averages chroma; this encoder (oracle/csc_ref.c matrix 1) sums each 2x2 box
and rounds once.  The two agree exactly on grey pictures (Y = v, Cb = Cr = 128 in both) and on pictures of 2x2-uniform blocks
whose colours convert identically in both (agreeing_palette).  libjpeg-turbo fills a partial MCU with DC-only dummy blocks
where this encoder replicates edges, so a size that is not a multiple of 16 is compared with libjpeg-turbo's file of the
edge-padded picture, its SOF size patched back to the visible one (padded_reference)."""
import cv2
import numpy as np

import oracle
from tests import synth


def coded(n):
    return (n + 15) & ~15


def libjpeg_420(bgr, quality):
    """libjpeg-turbo's baseline 4:2:0 JFIF file of a (H, W, 3) BGR picture (the first three channels of BGRA are used)."""
    ok, data = cv2.imencode(".jpg", np.ascontiguousarray(bgr[..., :3]), [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                                                        cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])
    assert ok
    return data.tobytes()


def segments(data):
    """[(marker, offset, length including the marker)] of the segments in front of the entropy-coded data, SOS last."""
    out, i = [], 2
    while True:
        assert data[i] == 0xFF, f"no marker at byte {i}"
        n = 2 + (data[i + 2] << 8 | data[i + 3])
        out.append((data[i + 1], i, n))
        if data[i + 1] == 0xDA:
            return out
        i += n


def patch_sof(data, w, h):
    d = bytearray(data)
    i = next(o for m, o, _ in segments(d) if m == 0xC0)
    d[i + 5: i + 9] = bytes((h >> 8, h & 255, w >> 8, w & 255))
    return bytes(d)


def padded_reference(bgr, w, h, quality):
    """libjpeg-turbo's file of `bgr` edge-padded to the coded size of a w x h picture, with SOF saying w x h.  `bgr` holds at
    least the w x h visible pixels and may already hold (part of) the padding."""
    cw, ch = coded(w), coded(h)
    p = bgr[:ch, :cw, :3]
    p = np.pad(p, ((0, ch - p.shape[0]), (0, cw - p.shape[1]), (0, 0)), mode="edge")
    return patch_sof(libjpeg_420(p, quality), w, h)


def stripe_reference(frame, y0, rows, quality):
    """What the stripe of `rows` picture rows from y0 of the JPEG mode must be: the rows of the picture edge-padded to its coded
    size, with SOF saying the stripe's visible rows (fewer than `rows` only for the last stripe, whose padding rows repeat the
    picture's last row)."""
    h, w = frame.shape[:2]
    return padded_reference(frame[y0: y0 + rows], w, min(rows, h - y0), quality)


def bgra(bgr):
    f = np.empty(bgr.shape[:2] + (4,), np.uint8)
    f[..., :3] = bgr
    f[..., 3] = 255
    return f


def grey(values):
    """BGRA picture whose three channels hold the (H, W) uint8 `values`."""
    return bgra(np.repeat(values[..., None], 3, 2))


def grey_noise(w, h, seed, binary=False):
    """Uniform grey noise, or (binary) noise of black and white pixels: the densest content found for this coder."""
    v = np.random.default_rng(seed).integers(0, 2 if binary else 256, (h, w))
    return grey((v * 255 if binary else v).astype(np.uint8))


def grey_desktop(w, h, t=0):
    return grey(np.rint(synth.desktop(w, h, t)[..., :3].mean(axis=2)).astype(np.uint8))


def agreeing_palette(rng, n):
    """Of n random colours, those whose flat 16x16 quality-100 file is the same from oracle.jpeg_encode_bgra and from
    libjpeg-turbo: at quality 100 every quantiser is 1, so the DC levels pin Y, Cb and Cr exactly.  (n, 3) BGR uint8."""
    keep = []
    for c in rng.integers(0, 256, (n, 3)).astype(np.uint8):
        f = bgra(np.broadcast_to(c, (16, 16, 3)))
        if oracle.jpeg_encode_bgra(f, 100) == libjpeg_420(f, 100):
            keep.append(c)
    return np.array(keep, np.uint8)


def mosaic(palette, w, h, seed):
    """BGRA picture of 2x2-uniform blocks of palette colours (w, h even): every chroma sample sees one colour."""
    idx = np.random.default_rng(seed).integers(0, len(palette), (h // 2, w // 2))
    return bgra(palette[idx].repeat(2, 0).repeat(2, 1))


def _huffman_tables(data):
    """{(class, id): {(length, code): symbol}} from the DHT segments."""
    tables = {}
    for m, o, n in segments(data):
        i = o + 4
        while m == 0xC4 and i < o + n:
            counts, i = data[i + 1: i + 17], i + 17
            t, code, k = {}, 0, 0
            for length, c in enumerate(counts, 1):
                for _ in range(c):
                    t[(length, code)] = data[i + k]
                    code, k = code + 1, k + 1
                code <<= 1
            tables[(data[i - 17] >> 4, data[i - 17] & 15)] = t
            i += k
    return tables


def _mcu_at(data, byte, mcus_per_row):
    """Index of the MCU of a 3-component 4:2:0 file whose coded bits contain scan byte `byte` (an offset into the file)."""
    start = sum(segments(data)[-1][1:])
    tables = _huffman_tables(data)
    unstuffed = bytearray()
    target = None
    i = start
    while i < len(data) - 2:
        if i >= byte and target is None:
            target = 8 * len(unstuffed)
        unstuffed.append(data[i])
        i += 2 if data[i] == 0xFF else 1
    bits = "".join(format(b, "08b") for b in unstuffed)
    pos = 0

    def symbol(t):
        nonlocal pos
        code = 0
        for length in range(1, 17):
            code, pos = 2 * code + int(bits[pos]), pos + 1
            if (length, code) in t:
                return t[(length, code)]
        raise ValueError(f"no Huffman code at bit {pos}")
    mcu = -1
    while pos <= (target if target is not None else len(bits)) and pos < len(bits) - 7:      # (the rest: padding)
        mcu += 1
        for tab in (0, 0, 0, 0, 1, 1):
            size = symbol(tables[(0, tab)])
            k, pos = 1, pos + size
            while k < 64:
                rs = symbol(tables[(1, tab)])
                if rs & 15 == 0 and rs != 0xF0:
                    break
                k, pos = k + (rs >> 4) + 1, pos + (rs & 15)
    return mcu, divmod(mcu, mcus_per_row)


def difference(got, want, width):
    """Where `got` first differs from the reference file `want` of a picture `width` pixels wide: the byte, and the header
    segment or the MCU (index, (row, column)) it falls in.  '' when the files are equal."""
    if got == want:
        return ""
    m = min(len(got), len(want))
    d = np.flatnonzero(np.frombuffer(got, np.uint8, m) != np.frombuffer(want, np.uint8, m))
    byte = int(d[0]) if d.size else m
    where = "past the end of the shorter file"
    segs = segments(want)
    for mk, o, n in segs:
        if o <= byte < o + n:
            where = f"in the header segment FF{mk:02X} at byte {o}"
    if byte >= sum(segs[-1][1:]):
        try:
            mcu, rc = _mcu_at(want, byte, coded(width) // 16)
            where = f"in MCU {mcu} (MCU row {rc[0]}, column {rc[1]})"
        except (ValueError, IndexError):
            where = "in the scan"
    return f"{len(got)} B against libjpeg-turbo's {len(want)} B; first difference at byte {byte}, {where}"
