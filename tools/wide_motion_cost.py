"""What B2V_FLAG_WIDE_MOTION buys and costs.

  bytes  (CPU, the oracle; by parity these are the GPU's bytes) bytes per P picture with the flag off and on, the mean over pictures
         2..5 of six: the desktop's text region scrolled at 8..250 px per picture (1080p, CQP 26) and window drags (720p, CQP 26).
  gpu    (H100) pictures/s through fresh sessions with the flag off and on, alternating, device-timed: bench.py's `value` workload (4K
         desktop scrolling 8 px per picture, CBR 20 Mbit/s at 60 fps nominal, 16 distinct frames resident in HBM, no callback) and
         the same with the text region scrolling 96 px per picture; then k_coarse's device time per picture (torch.profiler, CUDA
         activities, in a run of its own) on the fast scroll.  The card's name and power limit are read in the same run.

    python tools/wide_motion_cost.py [--part bytes|gpu|all] [--runs 5] [--pictures 512] [--out FILE.json]   (JSON printed either way)"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import synth                        # noqa: E402
from tests import wide_content as WC           # noqa: E402

W, H, FPS, KBPS, DISTINCT = 3840, 2160, 60.0, 20000, 16
SCROLLS = (8, 16, 17, 24, 40, 64, 96, 128, 250)
DRAGS = ((40, -30), (-100, 0), (127, 60))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def bytes_part() -> dict:
    import oracle
    from oracle.wide import WideRefEncoder
    oracle.set_threads(0)

    def p_bytes(frames, wide, w, h):
        e = WideRefEncoder(w, h)
        e.set_wide_motion(wide)
        sizes = [len(e.encode_bgra(f, k == 0, rc_mode=1, qp=26)) for k, f in enumerate(frames)]
        return int(statistics.mean(sizes[2:]))

    out = {"scroll_1080p_qp26": {}, "drag_720p_qp26": {}}
    for s in SCROLLS:
        frames = [WC.desktop_scroll(1920, 1080, t, s) for t in range(6)]
        r = {"off": p_bytes(frames, False, 1920, 1080), "on": p_bytes(frames, True, 1920, 1080)}
        r["on_over_off"] = r["on"] / r["off"]
        out["scroll_1080p_qp26"][f"{s}px"] = r
        print(json.dumps({f"scroll {s}px": r}), flush=True)
    for v in DRAGS:
        start = (560 - 2 * v[0], 240 - 2 * v[1])
        frames = [WC.drag(1280, 720, t, v, start) for t in range(6)]
        r = {"off": p_bytes(frames, False, 1280, 720), "on": p_bytes(frames, True, 1280, 720)}
        r["on_over_off"] = r["on"] / r["off"]
        out["drag_720p_qp26"][f"{v[0]},{v[1]}"] = r
        print(json.dumps({f"drag {v}": r}), flush=True)
    return out


def gpu_part(runs: int, pictures: int, warm: int) -> dict:
    from selkies_b200 import _native as N
    from selkies_b200.session import Session
    contents = {"desktop_8px": [synth.desktop(W, H, t) for t in range(DISTINCT)],
                "text_scroll_96px": [WC.desktop_scroll(W, H, t, 96) for t in range(DISTINCT)]}

    def session(frames, wide: bool):
        s = Session(W, H, fps=FPS, rc_mode=N.B2V_RC_CBR, bitrate_kbps=KBPS, ring_slots=DISTINCT, collect=False, wide_motion=wide)
        for i, f in enumerate(frames):
            s.resident_upload(i, f)
        return s

    def rate(frames, wide: bool) -> float:
        with session(frames, wide) as s:
            for k in range(warm):
                s.submit_resident(k % DISTINCT)
            s.timer_start()
            for k in range(pictures):
                s.submit_resident((warm + k) % DISTINCT)
            ms = s.timer_stop()
        return pictures / (ms / 1000.0)

    out = {"card": card(), "workload": f"{W}x{H} CBR {KBPS} kbit/s @ {FPS:g} fps nominal, {DISTINCT} resident frames cycled, no callback"}
    for name, frames in contents.items():
        off, on = [], []
        for _ in range(runs):
            off.append(rate(frames, False))
            on.append(rate(frames, True))
            print(json.dumps({name: {"off": off[-1], "on": on[-1]}}), flush=True)
        out[f"pictures_per_s_{name}"] = {"off": off, "on": on, "off_median": statistics.median(off), "on_median": statistics.median(on),
                                         "on_over_off": statistics.median(on) / statistics.median(off)}
    import torch
    from torch.profiler import ProfilerActivity, profile
    for name, frames in contents.items():
        with session(frames, True) as s:
            for k in range(warm):
                s.submit_resident(k % DISTINCT)
            s.flush()
            n = 4 * DISTINCT
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for k in range(n):
                    s.submit_resident(k % DISTINCT)
                s.flush()
                torch.cuda.synchronize()
        ev = [e for e in prof.events() if "k_coarse" in e.name]
        us = [e.device_time for e in ev] if ev and hasattr(ev[0], "device_time") else [e.cuda_time for e in ev]
        out[f"k_coarse_us_per_picture_{name}"] = {"n": len(us), "mean": statistics.mean(us) if us else None,
                                                   "max": max(us) if us else None}
        print(json.dumps({name: out[f"k_coarse_us_per_picture_{name}"]}), flush=True)
    out["card_after"] = card()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", choices=("bytes", "gpu", "all"), default="all")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--pictures", type=int, default=512)
    ap.add_argument("--warm", type=int, default=64)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    out = {}
    if a.part in ("bytes", "all"):
        out["bytes_per_p_picture"] = bytes_part()
    if a.part in ("gpu", "all"):
        out["gpu"] = gpu_part(a.runs, a.pictures, a.warm)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
