"""CPU-only checks of the drop-in boundary: the C-ABI library exports every symbol include/b2video.h declares,
the product never touches oracle/, and the Python mirror keeps the reference's interface."""
import ast
import asyncio
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "b2video.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2v_[a-z0-9_]+)\s*\(", src)) - {"b2v_cb"})


def test_library_exports_every_declared_symbol_at_abi_4():
    from selkies_b200 import _native
    lib = ctypes.CDLL(_native.LIB_PATH)
    declared = header_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/b2video.h but not exported"
    bound = {n for n, _, _ in _native.SYMBOLS}
    assert set(declared) == bound, set(declared) ^ bound
    header_abi = re.search(r"#define\s+B2V_ABI_VERSION\s+(\d+)", open(os.path.join(ROOT, "include", "b2video.h")).read())
    assert header_abi and int(header_abi.group(1)) == 4
    assert _native.lib().b2v_abi_version() == 4          # no compute call: safe without a GPU


def test_struct_layouts_match_header():
    from selkies_b200 import _native as N
    assert ctypes.sizeof(N.B2VSettings) == 4 * 4 + 8 + 14 * 4               # 80 bytes, a multiple of 8
    assert ctypes.sizeof(N.B2VFrame) == 8 + 4 * 4 + 8 + 8 + 2 * 4 and N.B2VFrame.y_start.offset == 40
    assert N.B2VSettings.fps.offset == 16 and N.B2VSettings.device.offset == 24
    assert ctypes.sizeof(N.B2VStats) == 7 * 8 + 7 * 8 + 6 * 8 + 2 * 8 + 8 * 8 and N.B2VStats.ns_wait_event.offset == 22 * 8


def test_product_never_imports_the_oracle():
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "selkies_b200")):
        for fn in files:
            p = os.path.join(dirpath, fn)
            if fn.endswith(".py"):
                tree = ast.parse(open(p).read())
                for node in ast.walk(tree):
                    names = []
                    if isinstance(node, ast.Import):
                        names = [a.name for a in node.names]
                    elif isinstance(node, ast.ImportFrom):
                        names = [node.module or ""]
                    bad += [(p, n) for n in names if n.split(".")[0] == "oracle"]
            elif fn.endswith((".cu", ".cuh", ".h", ".cpp")) or fn == "Makefile":
                if re.search(r'#include\s*"[^"]*oracle|\.\./\.\./oracle|liboracle', open(p).read()):
                    bad.append((p, "oracle reference"))
    assert not bad, bad


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from selkies_b200 import _native
    monkeypatch.setattr(_native, "_lib", None)
    monkeypatch.setattr(_native, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(ImportError):
        _native.lib()


def test_media_pipeline_interface_matches_reference():
    """The ten abstract methods of src/selkies/media_pipeline.py:41-80."""
    from selkies_b200.media_pipeline import MediaPipeline, MediaPipelineB200, RateControlMode
    want = {"start_media_pipeline", "stop_media_pipeline", "is_media_pipeline_running", "set_pointer_visible", "set_framerate",
            "set_video_bitrate", "set_audio_bitrate", "dynamic_idr_frame", "update_rate_control_mode", "set_crf"}
    assert set(MediaPipeline.__abstractmethods__) == want
    assert not getattr(MediaPipelineB200, "__abstractmethods__", None)
    assert RateControlMode.CBR == "cbr" and RateControlMode.CRF == "crf"


def test_capture_settings_contract():
    from selkies_b200.pixelflux_compat import CaptureSettings, StripeCallback
    cs = CaptureSettings()
    for f in ("capture_width", "capture_height", "capture_x", "capture_y", "target_fps", "capture_cursor", "output_mode",
              "auto_adjust_screen_capture_size", "h264_streaming_mode", "h264_fullframe", "h264_fullcolor", "h264_crf",
              "h264_paintover_crf", "h264_paintover_burst_frames", "h264_cbr_mode", "h264_bitrate_kbps",
              "vaapi_render_node_index", "use_cpu", "jpeg_quality", "paint_over_jpeg_quality", "use_paint_over_quality",
              "paint_over_trigger_frames", "damage_block_threshold", "damage_block_duration", "scale", "debug_logging",
              "watermark_path", "watermark_location_enum"):
        assert hasattr(cs, f), f
    cs.some_future_field = 3                     # unknown fields must not raise
    assert StripeCallback(lambda p, u: 7)(None, None) == 7
    with pytest.raises(TypeError):
        StripeCallback(5)


class FakeCapture:
    """Stands in for the native module, the way a fake pixelflux would for the reference."""
    instances = []

    def __init__(self, source=None):
        self.calls, self.cb, self.settings = [], None, None
        FakeCapture.instances.append(self)

    def start_capture(self, settings, cb):
        self.settings, self.cb = settings, cb
        self.calls.append("start")

    def stop_capture(self):
        self.calls.append("stop")

    def update_framerate(self, f):
        self.calls.append(("fps", f))

    def update_video_bitrate(self, k):
        self.calls.append(("kbps", k))

    def request_idr_frame(self):
        self.calls.append("idr")

    def update_resolution(self, w, h):
        self.calls.append(("res", w, h))


def test_media_pipeline_host_logic(monkeypatch):
    import selkies_b200.media_pipeline as mp
    from selkies_b200.pixelflux_compat import _Result, _ResultPtr
    monkeypatch.setattr(mp, "ScreenCapture", FakeCapture)
    FakeCapture.instances.clear()

    async def scenario():
        loop = asyncio.get_running_loop()
        got = []
        p = mp.MediaPipelineB200(loop, "x264enc", framerate=30, video_bitrate=8, width=1280, height=720, crf=23)

        async def produce(buf, pts, kind):
            got.append((buf, pts, kind))
        p.produce_data = produce
        await p.set_framerate(60)                 # not running: ignored
        await p.start_media_pipeline()
        assert p.is_media_pipeline_running()
        cap = FakeCapture.instances[-1]
        cs = cap.settings
        assert (cs.capture_width, cs.capture_height, cs.target_fps, cs.output_mode) == (1280, 720, 30.0, 1)
        assert cs.h264_cbr_mode is True and cs.h264_bitrate_kbps == 8000 and cs.h264_crf == 23 and cs.use_cpu is True
        # callback: 10-byte header stripped, pts = frame_id * (90000 // fps)
        r = _Result()
        r.data = memoryview(bytes(range(10)) + b"\x00\x00\x00\x01payload")
        r.size, r.frame_id = len(r.data), 7
        cap.cb(_ResultPtr(r), None)
        cap.cb(None, None)                        # falsy pointer ignored
        await asyncio.sleep(0.05)
        assert got == [(b"\x00\x00\x00\x01payload", 7 * 3000, "video")]
        await p.set_video_bitrate(8)              # unchanged: ignored
        await p.set_video_bitrate(0)              # <= 0: ignored
        await p.set_video_bitrate(20)             # Mbps -> kbps
        await p.set_framerate(30)                 # unchanged
        await p.set_framerate(-1)
        await p.set_framerate(60)
        await p.dynamic_idr_frame()
        await p.set_crf(30)                       # CBR mode: ignored
        assert cap.calls == ["start", ("kbps", 20000), ("fps", 60.0), "idr"]
        r.frame_id = 2
        cap.cb(_ResultPtr(r), None)
        await asyncio.sleep(0.05)
        assert got[-1][1] == 2 * 1500             # the pts step follows the new framerate
        await p.update_rate_control_mode(mp.RateControlMode.CRF)     # restart with new settings
        cap2 = FakeCapture.instances[-1]
        assert cap.calls[-1] == "stop" and cap2 is not cap and cap2.settings.h264_cbr_mode is False
        await p.set_video_bitrate(30)             # CRF mode: ignored
        await p.set_crf(30)
        cap3 = FakeCapture.instances[-1]
        assert cap3.settings.h264_crf == 30
        await p.set_resolution(1921, 1081)        # rounds down to even
        assert (p.width, p.height) == (1920, 1080) and cap3.calls[-1] == ("res", 1920, 1080)
        await p.stop_media_pipeline()
        assert not p.is_media_pipeline_running() and cap3.calls[-1] == "stop"

    asyncio.run(scenario())


def test_session_sharding_rule():
    from selkies_b200.multi_gpu import session_device
    assert [session_device(i, 8) for i in range(10)] == [0, 1, 2, 3, 4, 5, 6, 7, 0, 1]
    with pytest.raises(ValueError):
        session_device(0, 0)


def test_c_abi_argument_errors_without_a_gpu():
    """Error behaviour of the boundary: bad arguments give B2V_EINVAL + a message, never a crash (no CUDA call is reached)."""
    import ctypes as C
    from selkies_b200 import _native as N
    lib = N.lib()
    h = C.c_void_p()
    s = N.B2VSettings()
    s.src_w, s.src_h, s.fps = 1921, 1080, 60.0                       # odd width
    assert lib.b2v_create(C.byref(s), N.FRAME_CB(lambda f, u: None), None, C.byref(h)) == N.B2V_EINVAL
    assert b"unsupported" in lib.b2v_last_error()
    s.src_w, s.src_h = 8192, 4320                                    # beyond 7680x4320 (selkies.py:281)
    assert lib.b2v_create(C.byref(s), N.FRAME_CB(lambda f, u: None), None, C.byref(h)) == N.B2V_EINVAL
    assert lib.b2v_create(None, N.FRAME_CB(lambda f, u: None), None, C.byref(h)) == N.B2V_EINVAL
    for fn, args in ((lib.b2v_flush, (None,)), (lib.b2v_request_idr, (None,)), (lib.b2v_set_framerate, (None, 30.0)),
                     (lib.b2v_set_bitrate_kbps, (None, 1000)), (lib.b2v_get_stats, (None, None))):
        assert fn(*args) == N.B2V_EINVAL
    lib.b2v_destroy(None)                                            # no-op
    n = C.c_int32()
    assert lib.b2v_rtp_h264_packetize(None, 0, 1300, None, 0, None, 0, C.byref(n)) == N.B2V_EINVAL
    with pytest.raises(N.B2VError):
        N.check(N.B2V_EINVAL)


def test_keyframe_distance_is_seconds():
    """settings.py:163: keyframe_distance is in seconds; b2v_settings.gop is in frames (ADVICE r1)."""
    from selkies_b200.pixelflux_compat import ScreenCapture
    assert ScreenCapture._gop_frames(-1, 60.0) == -1
    assert ScreenCapture._gop_frames(0, 60.0) == -1
    assert ScreenCapture._gop_frames(2, 60.0) == 120
    assert ScreenCapture._gop_frames(1, 30.0) == 30
    assert ScreenCapture._gop_frames(0.001, 30.0) == 1
