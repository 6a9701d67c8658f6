"""oracle/h264_tables_ref.h vs the copy of the H.264 CAVLC tables compiled into libavcodec's decoder."""
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def parse_tables(path):
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for m in re.finditer(r"static const uint\d+_t (\w+)((?:\[\d+\])+)\s*=\s*\{(.*?)\};", src, flags=re.S):
        name, dims, body = m.group(1), [int(d) for d in re.findall(r"\[(\d+)\]", m.group(2))], m.group(3)
        if len(dims) == 1:
            out[name] = [int(v) for v in re.findall(r"-?\d+", body)]
        else:
            rows = re.findall(r"\{([^{}]*)\}", body)
            out[name] = [([int(v) for v in re.findall(r"-?\d+", r)] + [0] * dims[1])[: dims[1]] for r in rows]
    return out


def libavcodec_bytes():
    cv2 = pytest.importorskip("cv2")
    d = os.path.join(os.path.dirname(os.path.dirname(cv2.__file__)), "opencv_python_headless.libs")
    files = glob.glob(os.path.join(d, "libavcodec-*.so*"))
    if not files:
        pytest.skip("no bundled libavcodec")
    return open(files[0], "rb").read()


@pytest.mark.parametrize("path", ["oracle/h264_tables_ref.h", "selkies_b200/csrc/h264_tables.cuh"])
def test_tables_match_libavcodec(path):
    full = os.path.join(ROOT, path)
    if not os.path.exists(full):
        pytest.skip(f"{path} not present")
    t = parse_tables(full)
    blob = libavcodec_bytes()
    flat = lambda rows: bytes(v for r in rows for v in r)
    # coeff_token: ffmpeg stores [4][4*17] exactly like ours
    assert blob.count(flat(t["coeff_token_len"])) >= 1
    assert blob.count(flat(t["coeff_token_bits"])) >= 1
    assert blob.count(bytes(t["chroma_dc_coeff_token_len"])) >= 1
    assert blob.count(bytes(t["chroma_dc_coeff_token_bits"])) >= 1
    # total_zeros: ffmpeg [16][16] with a leading unused row? it stores 15 rows of 16
    assert blob.count(flat(t["total_zeros_len"])) >= 1
    assert blob.count(flat(t["total_zeros_bits"])) >= 1
    assert blob.count(flat(t["chroma_dc_total_zeros_len"])) >= 1
    assert blob.count(flat(t["chroma_dc_total_zeros_bits"])) >= 1
    assert blob.count(flat(t["run_len"])) >= 1
    assert blob.count(flat(t["run_bits"])) >= 1
    # coded_block_pattern mapping: ours is codeNum[cbp]; ffmpeg stores cbp[codeNum]
    for ours, theirs_prefix in (("cbp_to_codenum_intra", [47, 31, 15, 0, 23, 27, 29, 30]), ("cbp_to_codenum_inter", [0, 16, 1, 2, 4, 8, 32, 3])):
        inv = [0] * 48
        for cbp, code in enumerate(t[ours]):
            inv[code] = cbp
        assert inv[:8] == theirs_prefix
        assert blob.count(bytes(inv)) >= 1
    assert sorted(t["zigzag4x4"]) == list(range(16))
    assert blob.count(bytes(t["chroma_qp_tab"])) >= 1


@pytest.mark.parametrize("path", ["oracle/h264_tables_ref.h", "selkies_b200/csrc/h264_tables.cuh"])
def test_lambda_tables_follow_the_model(path):
    """The encoders' λ tables are the ones tests/h264_model.py states: the motion λ table, and rd_lambda of the intra decision
    (DESIGN.md §5.2), round(0.85·2^((qp − 12)/3)) and at least 1, which the model derives from the formula."""
    from tests import h264_model as M
    t = parse_tables(os.path.join(ROOT, path))
    assert t["me_lambda"] == M.LAMBDA
    assert t["rd_lambda"] == [M.rd_lambda(qp) for qp in range(52)]
