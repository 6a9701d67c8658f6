"""GPU time per picture with B2V_FLAG_SIZE_CAP off and on (cap 0, so nothing is recoded, and a cap that recodes the large pictures),
for steady content and for a scroll restart at 1080p and 4K, CQP 26, resident frames.  The time is the host clock around a submit
loop that ends in b2v_flush, over `--steps` pictures after `--warmup`, the variants alternated `--repeats` times; the median is
reported with the spread (max - min) of the repeats.  With the flag, entropy coding runs on the analysis stream: the "cap 0" column
is that cost as measured.  For every variant an untimed pass over the same cycle counts the P pictures coded above QP 26 (recoded).
Prints the card's name and power limit with the numbers and writes them as JSON (--out)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from selkies_b200 import _native as N  # noqa: E402
from selkies_b200.session import Session  # noqa: E402
from tests import synth  # noqa: E402


def contents(w, h):
    still = synth.desktop(w, h, 0)
    return {"steady": [synth.desktop(w, h, t) for t in range(8)],          # the text region scrolls 8 px per picture
            "scroll_restart": [still] * 4 + [synth.desktop(w, h, t) for t in range(1, 5)]}


def per_picture_ms(w, h, frames, flags, cap, steps, warmup):
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=26, flags=flags, collect=False) as s:
        if cap:
            s.set_max_picture_bytes(cap)
        for k, f in enumerate(frames):
            s.resident_upload(k, f)
        for i in range(warmup):
            s.submit_resident(i % len(frames))
        s.flush()
        t0 = time.perf_counter()
        for i in range(steps):
            s.submit_resident(i % len(frames))
        s.flush()
        return (time.perf_counter() - t0) * 1000.0 / steps


def recoded(w, h, frames, flags, cap, n):
    """P pictures coded above the session's QP 26 among n pictures of the cycle (the first, an IDR, excluded)."""
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=26, flags=flags) as s:
        if cap:
            s.set_max_picture_bytes(cap)
        for k, f in enumerate(frames):
            s.resident_upload(k, f)
        for i in range(n):
            s.submit_resident(i % len(frames))
        s.flush()
        got = s.take_frames()
    return sum(1 for x in got[1:] if x.qp > 26), len(got) - 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=240)
    ap.add_argument("--warmup", type=int, default=24)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", card)
    variants = {"off": (0, 0), "cap 0": (N.B2V_FLAG_SIZE_CAP, 0)}
    rows = []
    for w, h, cap in ((1920, 1080, 20000), (3840, 2160, 60000)):
        vs = dict(variants, **{f"cap {cap}": (N.B2V_FLAG_SIZE_CAP, cap)})
        for name, frames in contents(w, h).items():
            t = {k: [] for k in vs}
            for _ in range(a.repeats):
                for k, (flags, c) in vs.items():
                    t[k].append(per_picture_ms(w, h, frames, flags, c, a.steps, a.warmup))
            med = {k: statistics.median(v) for k, v in t.items()}
            spread = {k: max(v) - min(v) for k, v in t.items()}
            rec = {k: recoded(w, h, frames, flags, c, 4 * len(frames)) for k, (flags, c) in vs.items()}
            rows.append(dict(size=f"{w}x{h}", content=name, ms=med, spread=spread, recoded=rec))
            print(f"{w}x{h} {name:<15} " + "  ".join(f"{k}: {med[k]:.3f} ms (spread {spread[k]:.3f}, recoded {rec[k][0]}/{rec[k][1]})"
                                                      for k in vs))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
