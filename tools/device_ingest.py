"""Device-frame ingest on one GPU: what b2v_submit_device costs next to b2v_submit_resident, and what the CSC kernels of each
pixel format reach.  Everything runs in one process on one card, whose name, power limit and SM clock are printed beside the
numbers.

  pictures/s  4K, 16 distinct desktop frames, the settings of bench.py's `value` leg (CBR 20 Mbit/s, 60 fps, 64-picture
              steps, device-timed): `resident` (the library's copy, b2v_submit_resident) against `device` (the same frames in
              torch tensors, b2v_submit_device on torch's current stream), --runs alternating runs of each; ranges reported.
  csc         ms per CSC launch at 4K and 8K for each format (B2V_FLAG_NO_ENCODE | B2V_FLAG_TIMING_CSC sessions fed device
              frames: a CUDA-event pair around every 4th launch), as a fraction of 3.35 TB/s (H100 SXM data sheet) for
              5.5 B/px (4-byte formats) or 4.5 B/px (3-byte formats); beside it the BGRA resident b2v_bench_csc_burst figure.
  unaligned   the same at 4K for a window whose origin is not 16-byte aligned (3 px, 1 row into a larger surface): the general
              kernel.

Usage: python tools/device_ingest.py [--device 0] [--steps 16] [--warmup 2] [--runs 5] [--out FILE.json]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H = 3840, 2160
FPS, KBPS, STEP, N_DISTINCT = 60.0, 20000, 64, 16
HBM_GBS = 3350.0
FORMATS = {"BGRA": 5.5, "RGBA": 5.5, "BGR": 4.5, "RGB": 4.5}      # algorithmic bytes per pixel: read + 1.5 B of NV12 written


def card(device: int) -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", str(device), f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError(f"nvidia-smi failed: {out.stderr.strip()}")
    return dict(zip(q.split(","), (v.strip() for v in out.stdout.strip().split(","))))


def throughput(frames, surfaces, device: int, steps: int, warmup: int) -> float:
    """Pictures/s of one fresh session: resident frames when `surfaces` is None, else device submits of the tensors."""
    from selkies_b200 import _native as N
    from selkies_b200.session import Session
    with Session(W, H, fps=FPS, device=device, rc_mode=N.B2V_RC_CBR, bitrate_kbps=KBPS, ring_slots=N_DISTINCT, collect=False) as s:
        if surfaces is None:
            for i, f in enumerate(frames):
                s.resident_upload(i, f)
            submit = lambda k: s.submit_resident(k % N_DISTINCT)         # noqa: E731
        else:
            submit = lambda k: s.submit_device(surfaces[k % N_DISTINCT])  # noqa: E731
        k = 0
        for _ in range(warmup * STEP):
            submit(k); k += 1
        s.flush()
        s.timer_start()
        for _ in range(steps * STEP):
            submit(k); k += 1
        ms = s.timer_stop()
    return steps * STEP / (ms / 1000.0)


def csc_ms(w, h, surfaces, fmt, device: int, origin=(0, 0), pictures: int = 512) -> float:
    """Mean ms per CSC launch (CUDA events around every 4th launch) of device submits of `surfaces`."""
    from selkies_b200 import _native as N
    from selkies_b200.session import Session
    with Session(w, h, device=device, flags=N.B2V_FLAG_NO_ENCODE | N.B2V_FLAG_TIMING_CSC, ring_slots=8, collect=False) as s:
        for k in range(64):
            s.submit_device(surfaces[k % len(surfaces)], pixel_format=fmt, origin=origin)
        s.flush()
        s.reset_stats()
        for k in range(pictures):
            s.submit_device(surfaces[k % len(surfaces)], pixel_format=fmt, origin=origin)
        s.flush()
        st = s.stats()
    return st["ms_csc"] / max(1, st["n_csc"])


def burst_ms(w, h, frames, device: int) -> float:
    from selkies_b200 import _native as N
    from selkies_b200.session import Session
    with Session(w, h, device=device, flags=N.B2V_FLAG_NO_ENCODE, collect=False) as s:
        for i, f in enumerate(frames):
            s.resident_upload(i, f)
        return s.bench_csc_burst(len(frames), 512)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import numpy as np
    import torch
    from tests import synth
    from tests.device_scenario import device_surface
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    dev = a.device
    torch.cuda.set_device(dev)
    res = {"card": card(dev)}
    print("card:", res["card"], flush=True)

    frames = [synth.desktop(W, H, t) for t in range(N_DISTINCT)]
    surfaces = [device_surface(f, "BGRA", device=dev) for f in frames]
    runs = {"resident": [], "device": []}
    for _ in range(a.runs):
        runs["resident"].append(throughput(frames, None, dev, a.steps, a.warmup))
        runs["device"].append(throughput(frames, surfaces, dev, a.steps, a.warmup))
    res["pictures_per_s"] = {k: {"runs": [round(v, 1) for v in r], "min": round(min(r), 1), "max": round(max(r), 1)} for k, r in runs.items()}
    print("4K pictures/s:", json.dumps(res["pictures_per_s"]), flush=True)
    del surfaces

    res["csc"] = []
    sizes = {"4K": (W, H, frames), "8K": (2 * W, 2 * H, [np.tile(f, (2, 2, 1)) for f in frames[:4]])}
    for name, (w, h, fr) in sizes.items():
        burst = burst_ms(w, h, fr, dev)
        row = {"size": name, "bgra_resident_burst_ms": round(burst, 4), "bgra_resident_burst_frac": round(w * h * 5.5 / (burst * 1e-3) / 1e9 / HBM_GBS, 3)}
        for fmt, bpp in FORMATS.items():
            sf = [device_surface(f, fmt, device=dev) for f in fr]
            ms = csc_ms(w, h, sf, fmt, dev)
            row[fmt] = {"ms": round(ms, 4), "frac": round(w * h * bpp / (ms * 1e-3) / 1e9 / HBM_GBS, 3)}
            if name == "4K":
                sfu = [device_surface(f, fmt, margin=(3, 1), device=dev) for f in fr]
                msu = csc_ms(w, h, sfu, fmt, dev, origin=(3, 1))
                row[fmt]["unaligned_ms"] = round(msu, 4)
                row[fmt]["unaligned_frac"] = round(w * h * bpp / (msu * 1e-3) / 1e9 / HBM_GBS, 3)
                del sfu
            del sf
            torch.cuda.empty_cache()
        res["csc"].append(row)
        print("csc:", json.dumps(row), flush=True)
    res["card_after"] = card(dev)
    res["time"] = time.strftime("%Y-%m-%d %H:%M:%S")
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
