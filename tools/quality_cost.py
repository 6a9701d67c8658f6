"""What B2V_FLAG_QUALITY costs: bench.py's `value` workload (4K desktop, CBR 20 Mbit/s at 60 fps nominal, 16 distinct frames
resident in HBM and cycled, no callback) through fresh sessions with the flag off and on, alternating, device-timed
(b2v_timer_start / b2v_timer_stop).  A separate run under torch.profiler gives k_quality's own kernel time, against the
3 bytes per pixel it has to read (S and R: 1.5 B/px each in NV12).

    python tools/quality_cost.py [--runs 5] [--pictures 512] [--out FILE.json]      (the JSON is printed either way)"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from selkies_b200 import _native as N          # noqa: E402
from selkies_b200.session import Session       # noqa: E402
from tests import synth                        # noqa: E402

W, H, FPS, KBPS, DISTINCT = 3840, 2160, 60.0, 20000, 16
HBM_PEAK_GBS = 3350.0                          # H100 SXM data sheet (HBM3, 700 W card)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def session(quality: bool, frames):
    s = Session(W, H, fps=FPS, rc_mode=N.B2V_RC_CBR, bitrate_kbps=KBPS, ring_slots=DISTINCT, collect=False, quality=quality)
    for i, f in enumerate(frames):
        s.resident_upload(i, f)
    return s


def timed(quality: bool, frames, pictures: int, warm: int) -> float:
    with session(quality, frames) as s:
        for k in range(warm):
            s.submit_resident(k % DISTINCT)
        s.timer_start()
        for k in range(pictures):
            s.submit_resident((warm + k) % DISTINCT)
        ms = s.timer_stop()
    return pictures / (ms / 1000.0)


def kernel_times(frames, pictures: int, warm: int) -> dict:
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with session(True, frames) as s:
        for k in range(warm):
            s.submit_resident(k % DISTINCT)
        s.flush()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in range(pictures):
                s.submit_resident((warm + k) % DISTINCT)
            s.flush()
            torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            per.setdefault(e.name, []).append(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total)
    return {name: {"count": len(v), "mean_us": sum(v) / len(v)} for name, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--pictures", type=int, default=512)
    ap.add_argument("--warm", type=int, default=64)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    frames = [synth.desktop(W, H, t) for t in range(DISTINCT)]
    out = {"card": card(), "workload": f"{W}x{H} CBR {KBPS} kbit/s @ {FPS:g} fps nominal, {DISTINCT} resident frames cycled, no callback"}
    off, on = [], []
    for _ in range(a.runs):
        off.append(timed(False, frames, a.pictures, a.warm))
        on.append(timed(True, frames, a.pictures, a.warm))
        print(json.dumps({"off": off[-1], "on": on[-1]}), flush=True)
    out["pictures_per_s"] = {"off": off, "on": on, "off_median": statistics.median(off), "on_median": statistics.median(on),
                             "on_over_off": statistics.median(on) / statistics.median(off)}
    kt = kernel_times(frames, 256, a.warm)
    q = next((v for k, v in kt.items() if "k_quality" in k), None)
    out["kernels_us"] = {k: v for k, v in sorted(kt.items(), key=lambda kv: -kv[1]["mean_us"] * kv[1]["count"])[:12]}
    if q:
        traffic = 3 * W * H                      # bytes the measurement must read: S and R, luma + chroma
        out["k_quality"] = {"mean_us": q["mean_us"], "bytes": traffic, "achieved_GBs": traffic / (q["mean_us"] * 1e3),
                            "share_of_3.35TBs": traffic / (q["mean_us"] * 1e3) / HBM_PEAK_GBS}
    out["card_after"] = card()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
