"""What B2V_FLAG_SCENE_CUT buys and costs.

  bytes  (CPU, the oracle; by parity these are the GPU's bytes) the table of include/b2video.h / INTEGRATION.md §13: for each pair of
         whole-screen contents at 1080p, CQP 26 and 36, the second picture's bytes as a P picture (flag off), as an IDR picture, and
         with the flag on, and whether the flag cut it.
  gpu    (H100) the time per picture through fresh sessions with the flag off and on, alternating, device-timed, at 1080p and 4K,
         CBR (8 and 20 Mbit/s at 60 fps nominal), resident frames cycled, no callback: on steady content (synth.desktop scrolling 8 px
         per picture: no picture is cut) and on cut content (four different screens in turn: every P picture is a switch, cut with the
         flag on).  The extra time per P picture is on minus off.  The card's name and power limit are read in the same run.

    python tools/scene_cut_cost.py [--part bytes|gpu|all] [--runs 5] [--pictures 512] [--out FILE.json]   (JSON printed either way)"""
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

DISTINCT = 16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def pairs(w, h):
    return {"desktop -> desktop inverted": (LC.desktop(w, h, 1), LC.desktop(w, h, 1, invert=True)),
            "synth.desktop -> synth.bars": (synth.desktop(w, h), synth.bars(w, h)),
            "synth.desktop -> synth.gradient": (synth.desktop(w, h), synth.gradient(w, h)),
            "synth.gradient -> synth.desktop": (synth.gradient(w, h), synth.desktop(w, h)),
            "synth.desktop(seed=1) -> synth.desktop(seed=2)": (synth.desktop(w, h, seed=1), synth.desktop(w, h, seed=2)),
            "synth.noise(0) -> synth.noise(1)": (synth.noise(w, h, 0), synth.noise(w, h, 1))}


def bytes_part() -> dict:
    import oracle
    from oracle.scut import SceneCutEncoder
    oracle.set_threads(0)
    w, h = 1920, 1080
    out = {}
    for qp in (26, 36):
        for name, (a, b) in pairs(w, h).items():
            sizes = []
            for cut in (False, True):
                e = SceneCutEncoder(w, h)
                e.set_scene_cut(cut)
                e.encode_bgra(a, True, rc_mode=1, qp=qp)
                sizes.append(len(e.encode_bgra(b, False, rc_mode=1, qp=qp)))
                state = e.scut_state() if cut else None
                e.close()
            e = SceneCutEncoder(w, h)
            intra = len(e.encode_bgra(b, True, rc_mode=1, qp=qp))
            e.close()
            r = {"p_bytes": sizes[0], "idr_bytes": intra, "idr_over_p": intra / sizes[0], "flag_on_bytes": sizes[1],
                 "cut": bool(state["cut"]), "cost_intra": state["cost_intra"], "cost_inter": state["cost_inter"]}
            out[f"qp{qp} {name}"] = r
            print(json.dumps({f"qp{qp} {name}": r}), flush=True)
    return out


def gpu_part(runs: int, pictures: int, warm: int) -> dict:
    from selkies_b200 import _native as N
    from selkies_b200.session import Session

    def session(w, h, kbps, frames, cut: bool):
        s = Session(w, h, fps=60.0, rc_mode=N.B2V_RC_CBR, bitrate_kbps=kbps, ring_slots=len(frames), collect=False, scene_cut=cut)
        for i, f in enumerate(frames):
            s.resident_upload(i, f)
        return s

    def ms_per_picture(w, h, kbps, frames, cut: bool) -> float:
        with session(w, h, kbps, frames, cut) as s:
            for k in range(warm):
                s.submit_resident(k % len(frames))
            s.timer_start()
            for k in range(pictures):
                s.submit_resident((warm + k) % len(frames))
            ms = s.timer_stop()
        return ms / pictures

    def cuts(w, h, kbps, frames) -> float:
        with Session(w, h, fps=60.0, rc_mode=N.B2V_RC_CBR, bitrate_kbps=kbps, ring_slots=len(frames), scene_cut=True) as s:
            for i, f in enumerate(frames):
                s.resident_upload(i, f)
            for k in range(2 * len(frames)):
                s.submit_resident(k % len(frames))
            s.flush()
            got = s.take_frames()[1:]
            return sum(fr.intra for fr in got) / len(got)

    out = {"card": card(), "workload": "CBR at 60 fps nominal, resident frames cycled, no callback; ms per picture, device-timed"}
    for w, h, kbps in ((1920, 1080, 8000), (3840, 2160, 20000)):
        contents = {"steady": [synth.desktop(w, h, t) for t in range(DISTINCT)],
                    "cut": [LC.desktop(w, h, 1), synth.bars(w, h), LC.desktop(w, h, 1, invert=True), synth.gradient(w, h)]}
        for name, frames in contents.items():
            off, on = [], []
            for _ in range(runs):
                off.append(ms_per_picture(w, h, kbps, frames, False))
                on.append(ms_per_picture(w, h, kbps, frames, True))
            key = f"{w}x{h} {name}"
            out[key] = {"ms_off": off, "ms_on": on, "ms_off_median": statistics.median(off), "ms_on_median": statistics.median(on),
                        "extra_ms_per_picture": statistics.median(on) - statistics.median(off),
                        "cut_fraction_on": cuts(w, h, kbps, frames)}
            print(json.dumps({key: out[key]}), flush=True)
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
        out["bytes"] = bytes_part()
    if a.part in ("gpu", "all"):
        out["gpu"] = gpu_part(a.runs, a.pictures, a.warm)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
