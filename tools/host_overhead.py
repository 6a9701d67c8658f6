"""Host cost of one submit (ctypes call + kernel launches + job hand-off), measured while the rings are empty so nothing blocks.
Run on the GPU box:  python tools/host_overhead.py"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import synth

W, H = 3840, 2160
frames = [synth.desktop(W, H, t) for t in range(4)]
for flags, name in ((0, "plain"), (N.B2V_FLAG_TIMING, "timing")):
    with Session(W, H, rc_mode=N.B2V_RC_CBR, bitrate_kbps=20000, ring_slots=8, flags=flags, collect=False, on_frame=lambda fptr: None) as s:
        for i, f in enumerate(frames):
            s.resident_upload(i, f)
        for k in range(32):
            s.submit_resident(k % 4)
        s.flush()
        per = []
        for rep in range(20):
            t0 = time.perf_counter()
            for k in range(6):
                s.submit_resident(k % 4)
            per.append((time.perf_counter() - t0) / 6)
            s.flush()
        print(name, "submit_resident host us/frame: median %.1f min %.1f" % (1e6 * float(np.median(per)), 1e6 * min(per)))
        t0 = time.perf_counter()
        for k in range(400):
            s.submit_resident(k % 4)
        s.flush()
        print(name, "steady fps", 400 / (time.perf_counter() - t0))
