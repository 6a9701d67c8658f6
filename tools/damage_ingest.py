"""Damage-rectangle ingest (B2V_FLAG_DAMAGE) on one GPU: what the host ring costs per picture when only the changed regions are
written, copied and converted, next to whole-frame submits.  Everything runs in one process on one card, whose name and power
limit are printed beside the numbers.

  sizes     4K (3840 x 2160) and 1080p
  contents  typing (a few glyph cells per picture), a scrolling pane of about a third of the screen (8 rows per picture), and a
            full-screen change (a new noise picture every time)
  legs      off     whole-frame submits, a session without the flag (one device buffer per ring slot)
            whole   whole-frame submits, a session with the flag (the one mirror, the copy ordered after the previous CSC)
            damage  damage submits: only the changed rectangles are written into the slot, copied and converted
  per leg   end-to-end pictures/s through Session.submit (the producer's write into the pinned slot included), h2d_bytes per
            picture, host us per submit (ns_submit), CSC ms per launch (B2V_FLAG_TIMING_CSC), the share of dirty tiles.
            Legs are interleaved, --runs times each; min / median / max reported.

Usage: python tools/damage_ingest.py [--device 0] [--pictures 96] [--warmup 16] [--runs 3] [--out FILE.json]"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = {"4K": (3840, 2160), "1080p": (1920, 1080)}
N_DISTINCT, FPS, KBPS = 16, 60.0, 20000


def card(device: int) -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", str(device), f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError(f"nvidia-smi failed: {out.stderr.strip()}")
    return dict(zip(q.split(","), (v.strip() for v in out.stdout.strip().split(","))))


def content(name: str, w: int, h: int):
    """N_DISTINCT frames that cycle, and the rectangles that changed from frame k - 1 (cyclically) to frame k."""
    from tests import synth
    from tests.damage_scenario import damage
    rng = np.random.default_rng(1)
    base = synth.desktop(w, h, 0)
    frames = []
    if name == "typing":                 # a line of glyphs typed and erased: up to two 7 x 11 cells change per picture
        y = h // 2
        for k in range(N_DISTINCT):
            f = base.copy()
            n = k if k < N_DISTINCT // 2 else N_DISTINCT - k
            for i in range(n):
                f[y:y + 11, 200 + 8 * i:207 + 8 * i, :3] = 20
            frames.append(f)
    elif name == "scroll":               # a pane of w/2 x 2h/3 at (w/4, h/6), its content 8 rows further down each picture
        tall = rng.integers(0, 2, (2 * h // 3 + 8 * N_DISTINCT, w // 2), dtype=np.uint8) * 200 + 20
        tall[8 * N_DISTINCT:] = tall[:2 * h // 3]          # the pane wraps seamlessly
        for k in range(N_DISTINCT):
            f = base.copy()
            f[h // 6:h // 6 + 2 * h // 3, w // 4:w // 4 + w // 2, :3] = tall[8 * k:8 * k + 2 * h // 3, :, None]
            frames.append(f)
    else:                                # full: every pixel new
        frames = [synth.noise(w, h, k) for k in range(N_DISTINCT)]
    rects = [damage(frames[k - 1], frames[k]) for k in range(N_DISTINCT)]
    return frames, rects


def dirty_share(w: int, h: int, rects) -> float:
    from selkies_b200 import _native as N
    from selkies_b200.session import normalize_rects
    m = np.zeros(((w + 15) // 16) * ((h + 15) // 16), np.uint8)
    arr, n = N.rect_array(normalize_rects(rects, w, h))
    return N.lib().b2v_damage_tiles(w, h, w, h, arr, n, m.ctypes.data) / m.size


def leg(kind: str, frames, rects, device: int, pictures: int, warmup: int) -> dict:
    from selkies_b200 import _native as N
    from selkies_b200.session import Session
    h, w = frames[0].shape[:2]
    with Session(w, h, fps=FPS, device=device, rc_mode=N.B2V_RC_CBR, bitrate_kbps=KBPS, collect=False,
                 flags=N.B2V_FLAG_TIMING_CSC, damage=kind != "off") as s:
        def submit(k):
            i = k % N_DISTINCT
            s.submit(frames[i], damage=rects[i] if kind == "damage" and k > 0 else None)
        for k in range(warmup):
            submit(k)
        s.flush()
        s.reset_stats()
        t0 = time.perf_counter()
        for k in range(warmup, warmup + pictures):
            submit(k)
        s.flush()
        dt = time.perf_counter() - t0
        st = s.stats()
    return {"fps": pictures / dt, "h2d_per_picture": st["h2d_bytes"] / pictures, "us_submit": st["ns_submit"] / pictures / 1e3,
            "ms_csc": st["ms_csc"] / max(1, st["n_csc"])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--pictures", type=int, default=96)
    ap.add_argument("--warmup", type=int, default=16)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    result = {"card_before": card(a.device), "legs": {}}
    print(json.dumps(result["card_before"]), flush=True)
    for size, (w, h) in SIZES.items():
        for name in ("typing", "scroll", "full"):
            frames, rects = content(name, w, h)
            share = statistics.mean(dirty_share(w, h, r) for r in rects)
            runs = {k: [] for k in ("off", "whole", "damage")}
            for _ in range(a.runs):                      # interleaved
                for kind in runs:
                    runs[kind].append(leg(kind, frames, rects, a.device, a.pictures, a.warmup))
            for kind, rs in runs.items():
                row = {m: [round(min(r[m] for r in rs), 4), round(statistics.median(r[m] for r in rs), 4), round(max(r[m] for r in rs), 4)]
                       for m in rs[0]}
                row["dirty_tiles"] = round(share, 4) if kind == "damage" else 1.0
                result["legs"][f"{size}/{name}/{kind}"] = row
                print(f"{size:6s} {name:7s} {kind:7s} " + "  ".join(f"{m} {v[0]:.4g}/{v[1]:.4g}/{v[2]:.4g}" for m, v in row.items() if m != "dirty_tiles")
                      + f"  dirty {row['dirty_tiles']:.3f}", flush=True)
    result["card_after"] = card(a.device)
    print(json.dumps(result["card_after"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
