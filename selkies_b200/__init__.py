"""selkies_b200 — the H100-native video-frame hot path behind the selkies video-pipeline surface.

Only what the hot path needs lives here:
  csrc/               hand-written sm_90a CUDA kernels + the C-ABI (include/b2video.h)
  _native.py          ctypes binding (no CPU fallback)
  pixelflux_compat.py CaptureSettings / ScreenCapture / StripeCallback (the module the reference imports)
  media_pipeline.py   MediaPipeline ABC + MediaPipelineB200 (mirror of src/selkies/media_pipeline.py)
  gst_webrtc_app.py   GSTWebRTCApp façade (build_video_pipeline / set_framerate / set_resolution / set_video_bitrate)
"""
__version__ = "0.1.0"
