"""Generate tests/golden/rtp_h264_golden.json from the UNMODIFIED reference packetiser.

Needs a checkout of the reference project: REF_ROOT=<selkies checkout> python tools/make_rtp_golden.py.  The reference module
src/selkies/webrtc/codecs/h264.py imports PyAV and sibling modules that are absent here, but its packetiser
(`H264Encoder._split_bitstream / _packetize / _packetize_fu_a / _packetize_stap_a`, h264.py:165-279) is pure
Python: the script stubs the unused imports, executes the reference file as-is and records, for a set of
access units, the exact RTP payload list `pack()` would return.
"""
import base64
import importlib.util
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.path.join(os.environ.get("REF_ROOT", "."), "src", "selkies", "webrtc", "codecs", "h264.py")


def load_reference():
    for name in ["av", "av.frame", "av.packet", "av.video", "av.video.codeccontext"]:
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["av"].VideoFrame = object
    sys.modules["av"].Packet = object
    sys.modules["av.frame"].Frame = object
    sys.modules["av.packet"].Packet = object
    sys.modules["av.video.codeccontext"].VideoCodecContext = object
    pkg = types.ModuleType("refpkg"); pkg.__path__ = []
    codecs = types.ModuleType("refpkg.codecs"); codecs.__path__ = []
    jb = types.ModuleType("refpkg.jitterbuffer"); jb.JitterFrame = object
    ms = types.ModuleType("refpkg.mediastreams"); ms.VIDEO_TIME_BASE = None; ms.convert_timebase = lambda *a: 0
    base = types.ModuleType("refpkg.codecs.base"); base.Decoder = object; base.Encoder = object
    for m in (pkg, codecs, jb, ms, base):
        sys.modules[m.__name__] = m
    spec = importlib.util.spec_from_file_location("refpkg.codecs.h264", REF)
    mod = importlib.util.module_from_spec(spec)
    sys.modules["refpkg.codecs.h264"] = mod
    spec.loader.exec_module(mod)          # the reference source, unmodified
    return mod


def access_units():
    import numpy as np
    import oracle
    from tests import synth
    out = []
    # real encoder output: IDR (SPS+PPS+slices), P pictures, many small slice NALs, a few NALs > 1300 bytes
    for (w, h, qp, sr, n) in [(160, 96, 30, 1, 3), (160, 96, 12, 100, 2), (320, 192, 22, 4, 2), (64, 48, 2, 2, 2)]:
        enc = oracle.RefEncoder(w, h, sr)
        for t in range(n):
            out.append(enc.encode_bgra(synth.desktop(w, h, t), t == 0, qp=qp))
    rng = np.random.default_rng(7)
    def nal(n, hdr=0x41, long=False):
        body = bytes(rng.integers(4, 256, n - 1, dtype=np.uint8))     # no start-code emulation inside
        return (b"\x00\x00\x00\x01" if long else b"\x00\x00\x01") + bytes([hdr]) + body
    # boundary sizes around PACKET_MAX (h264.py:58), STAP-A count limit (9), nri propagation, trailing data
    out.append(nal(1300) + nal(1301) + nal(1299, 0x65, True))
    out.append(b"".join(nal(20 + i, 0x01 if i % 2 else 0x61) for i in range(14)))
    out.append(nal(2599) + nal(2600) + nal(2601) + nal(5, 0x67, True) + nal(4, 0x68, True))
    out.append(nal(1296) + nal(2) + nal(1297) + nal(1) + nal(3900, 0x25))
    out.append(b"")
    out.append(b"\x01\x02\x03 no start code at all")
    out.append(nal(600) + nal(600) + nal(600) + nal(97) + nal(1300))
    return out


def main():
    ref = load_reference()
    cases = []
    for au in access_units():
        payloads = ref.H264Encoder._packetize(ref.H264Encoder._split_bitstream(au))
        import hashlib
        cases.append({"au": base64.b64encode(au).decode(), "lens": [len(p) for p in payloads],
                      "sha256": [hashlib.sha256(p).hexdigest()[:24] for p in payloads],
                      "first": [base64.b64encode(p[:8]).decode() for p in payloads]})
    path = os.path.join(ROOT, "tests", "golden", "rtp_h264_golden.json")
    json.dump({"source": "selkies @1a9cd02b src/selkies/webrtc/codecs/h264.py:165-279 (H264Encoder._packetize), PACKET_MAX=1300",
               "cases": cases}, open(path, "w"))
    print(path, len(cases), "cases", os.path.getsize(path), "bytes", sum(len(c["lens"]) for c in cases), "packets")


if __name__ == "__main__":
    main()
