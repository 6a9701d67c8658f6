"""Short 4K run of the headline workload, as a target for a profiler:
python tools/profile_target.py [n_pictures] [gop]   — CBR 20 Mbit/s, inputs resident, two-stream schedule as in bench.py."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from selkies_b200 import _native as N          # noqa: E402
from selkies_b200.session import Session        # noqa: E402
from tests import synth                         # noqa: E402

W, H, ND = 3840, 2160, 16
n = int(sys.argv[1]) if len(sys.argv) > 1 else 48
gop = int(sys.argv[2]) if len(sys.argv) > 2 else -1
CONTENT = os.environ.get("B2V_CONTENT", "desktop")      # desktop (headline) | gradient (S4) | noise (S2)
frames = [{"desktop": synth.desktop, "gradient": synth.gradient}[CONTENT](W, H, t) if CONTENT != "noise" else synth.noise(W, H, 100 + t) for t in range(ND)]
with Session(W, H, fps=60.0, rc_mode=N.B2V_RC_CBR, bitrate_kbps=20000, ring_slots=4, gop=gop, collect=False) as s:
    for i, f in enumerate(frames):
        s.resident_upload(i, f)
    for k in range(n):
        s.submit_resident(k % ND)
    s.flush()
