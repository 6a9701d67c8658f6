"""What B2V_FLAG_DROPPABLE costs, per content and per layer.

  bytes  (CPU, the oracle; by parity these are the GPU's bytes) bytes per P picture with the flag off and on, split by the picture's
         count from the IDR: odd counts are the non-reference pictures with the flag (distance 1 to their reference), even counts
         the reference P pictures (distance 2).  Without the flag both kinds are ordinary P pictures at distance 1.
  gpu    (H100) bench.py's `value` workload (4K desktop scrolling 8 px per picture, CBR 20 Mbit/s at 60 fps nominal, 16 distinct
         frames resident in HBM, no callback) through fresh sessions with the flag off and on, alternating, device-timed; then
         ms_inter (B2V_FLAG_TIMING: the P-picture analysis, CUDA events) per picture, split by layer as above.  The card's name and
         power limit are read in the same run.

    python tools/droppable_cost.py [--part bytes|gpu|all] [--runs 5] [--pictures 512] [--out FILE.json]   (JSON printed either way)"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import synth                        # noqa: E402

W, H, FPS, KBPS, DISTINCT = 3840, 2160, 60.0, 20000, 16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def _by_layer(values):
    """values[k] of picture k (picture 0 the IDR) -> means over the P pictures at odd and at even counts."""
    odd, even = values[1::2], values[2::2]
    return {"odd": statistics.mean(odd), "even": statistics.mean(even), "all_p": statistics.mean(values[1:]), "n": len(values) - 1}


CONTENTS = {
    # name: (width, height, frames of picture k, oracle keywords)
    "desktop_scroll_8px_4k_qp28": (3840, 2160, lambda w, h, k: synth.desktop(w, h, k % DISTINCT), dict(rc_mode=1, qp=28)),
    "desktop_scroll_8px_1080p_qp28": (1920, 1080, lambda w, h, k: synth.desktop(w, h, k), dict(rc_mode=1, qp=28)),
    "gradient_pan_2px_1080p_qp28": (1920, 1080, lambda w, h, k: synth.gradient(w, h, k), dict(rc_mode=1, qp=28)),
    "bars_moving_box_1080p_qp28": (1920, 1080, lambda w, h, k: synth.bars(w, h, k), dict(rc_mode=1, qp=28)),
}


def bytes_part(pictures: int) -> dict:
    import oracle
    from oracle.layers import LayeredRefEncoder
    oracle.set_threads(0)
    out = {}
    for name, (w, h, frame, kw) in CONTENTS.items():
        res = {}
        for on in (False, True):
            e = LayeredRefEncoder(w, h)
            e.set_droppable(on)
            sizes = [len(e.encode_bgra(frame(w, h, k), k == 0, **kw)) for k in range(pictures)]
            res["on" if on else "off"] = _by_layer(sizes)
        res["on_over_off"] = {k: res["on"][k] / res["off"][k] for k in ("odd", "even", "all_p")}
        out[name] = res
        print(json.dumps({name: res}), flush=True)
    return out


def gpu_part(runs: int, pictures: int, warm: int) -> dict:
    from selkies_b200 import _native as N
    from selkies_b200.session import Session
    frames = [synth.desktop(W, H, t) for t in range(DISTINCT)]

    def session(on: bool, flags: int = 0):
        s = Session(W, H, fps=FPS, rc_mode=N.B2V_RC_CBR, bitrate_kbps=KBPS, ring_slots=DISTINCT, collect=False, droppable=on,
                    flags=flags)
        for i, f in enumerate(frames):
            s.resident_upload(i, f)
        return s

    def rate(on: bool) -> float:
        with session(on) as s:
            for k in range(warm):
                s.submit_resident(k % DISTINCT)
            s.timer_start()
            for k in range(pictures):
                s.submit_resident((warm + k) % DISTINCT)
            ms = s.timer_stop()
        return pictures / (ms / 1000.0)

    def inter_ms(on: bool, n: int) -> list:
        """ms_inter of pictures 0..n-1 (picture 0, the IDR, has none), one picture at a time."""
        per = []
        with session(on, N.B2V_FLAG_TIMING) as s:
            for k in range(n):
                before = s.stats()["ms_inter"]
                s.submit_resident(k % DISTINCT)
                s.flush()
                per.append(s.stats()["ms_inter"] - before)
        return per

    out = {"card": card(), "workload": f"{W}x{H} CBR {KBPS} kbit/s @ {FPS:g} fps nominal, {DISTINCT} resident frames cycled, no callback"}
    off, on = [], []
    for _ in range(runs):
        off.append(rate(False))
        on.append(rate(True))
        print(json.dumps({"off": off[-1], "on": on[-1]}), flush=True)
    out["pictures_per_s"] = {"off": off, "on": on, "off_median": statistics.median(off), "on_median": statistics.median(on),
                             "on_over_off": statistics.median(on) / statistics.median(off)}
    n = 4 * DISTINCT + 1                           # the IDR and 64 P pictures: four scroll cycles, restarts included
    inter_ms(False, 8)                             # warm-up: module load, first launches
    out["ms_inter_per_picture"] = {"off": _by_layer(inter_ms(False, n)), "on": _by_layer(inter_ms(True, n))}
    out["card_after"] = card()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", choices=("bytes", "gpu", "all"), default="all")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--pictures", type=int, default=512)
    ap.add_argument("--warm", type=int, default=64)
    ap.add_argument("--byte-pictures", type=int, default=33, help="pictures per content in the byte count (the IDR included)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    out = {}
    if a.part in ("bytes", "all"):
        out["bytes_per_picture"] = bytes_part(a.byte_pictures)
    if a.part in ("gpu", "all"):
        out["gpu"] = gpu_part(a.runs, a.pictures, a.warm)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
