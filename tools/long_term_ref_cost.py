"""What B2V_FLAG_LONG_TERM_REF buys and costs.

  bytes  (CPU, the oracle; by parity these are the GPU's bytes) bytes per picture with the flag off and on on the scripted contents
         of tests/ltr_content.py (1080p, CQP 26): the whole stream, and the pictures on which earlier content comes back (the
         popup closes, the switch back to an application).
  gpu    (H100) pictures/s through fresh sessions with the flag off and on, alternating, device-timed: bench.py's `value` workload
         (4K desktop scrolling 8 px per picture, CBR 20 Mbit/s at 60 fps nominal, 16 distinct frames resident in HBM, no callback)
         and the same on the 4K alt-tab content cycled (a reveal every third picture); bytes per picture of each from the
         sessions' own access units in a run of their own.  The card's name and power limit are read in the same run.

    python tools/long_term_ref_cost.py [--part bytes|gpu|all] [--runs 5] [--pictures 512] [--out FILE.json]   (JSON printed either way)"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import ltr_content as LC            # noqa: E402
from tests import synth                        # noqa: E402

W, H, FPS, KBPS, DISTINCT = 3840, 2160, 60.0, 20000, 16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def bytes_part() -> dict:
    import oracle
    from oracle.ltr import LongTermRefEncoder
    oracle.set_threads(0)

    def sizes(frames, ltr, w, h):
        e = LongTermRefEncoder(w, h)
        e.set_long_term_ref(ltr)
        return [len(e.encode_bgra(f, k == 0, rc_mode=1, qp=26)) for k, f in enumerate(frames)]

    out = {}
    for name, fn in sorted(LC.CONTENTS.items()):
        frames, returns = fn(1920, 1080)
        off, on = sizes(frames, False, 1920, 1080), sizes(frames, True, 1920, 1080)
        r = {"total_off": sum(off), "total_on": sum(on), "total_on_over_off": sum(on) / sum(off),
             "returns": {str(k): {"off": off[k], "on": on[k], "on_over_off": on[k] / off[k]} for k in returns}}
        out[name] = r
        print(json.dumps({name: r}), flush=True)
    return out


def gpu_part(runs: int, pictures: int, warm: int) -> dict:
    from selkies_b200 import _native as N
    from selkies_b200.session import Session
    contents = {"desktop_8px": [synth.desktop(W, H, t) for t in range(DISTINCT)], "alt_tab": LC.alt_tab(W, H)[0]}

    def session(frames, ltr: bool, collect=False):
        s = Session(W, H, fps=FPS, rc_mode=N.B2V_RC_CBR, bitrate_kbps=KBPS, ring_slots=DISTINCT, collect=collect, long_term_ref=ltr)
        for i, f in enumerate(frames):
            s.resident_upload(i, f)
        return s

    def rate(frames, ltr: bool) -> float:
        with session(frames, ltr) as s:
            for k in range(warm):
                s.submit_resident(k % len(frames))
            s.timer_start()
            for k in range(pictures):
                s.submit_resident((warm + k) % len(frames))
            ms = s.timer_stop()
        return pictures / (ms / 1000.0)

    def mean_bytes(frames, ltr: bool) -> float:
        with session(frames, ltr, collect=True) as s:
            for k in range(4 * len(frames)):
                s.submit_resident(k % len(frames))
            s.flush()
            return statistics.mean(len(fr.data) for fr in s.take_frames()[len(frames):])

    out = {"card": card(), "workload": f"{W}x{H} CBR {KBPS} kbit/s @ {FPS:g} fps nominal, resident frames cycled, no callback"}
    for name, frames in contents.items():
        off, on = [], []
        for _ in range(runs):
            off.append(rate(frames, False))
            on.append(rate(frames, True))
            print(json.dumps({name: {"off": off[-1], "on": on[-1]}}), flush=True)
        out[f"pictures_per_s_{name}"] = {"off": off, "on": on, "off_median": statistics.median(off), "on_median": statistics.median(on),
                                         "on_over_off": statistics.median(on) / statistics.median(off)}
        out[f"bytes_per_picture_{name}"] = {"off": mean_bytes(frames, False), "on": mean_bytes(frames, True)}
        print(json.dumps({name: out[f"bytes_per_picture_{name}"]}), flush=True)
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
        out["bytes_per_picture"] = bytes_part()
    if a.part in ("gpu", "all"):
        out["gpu"] = gpu_part(a.runs, a.pictures, a.warm)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
