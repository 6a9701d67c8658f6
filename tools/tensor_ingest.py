"""Tensor ingest on one GPU: what b2v_submit_tensor costs next to the preparation a user writes in front of b2v_submit_device,
and what the colour conversion reaches on each element type.  Everything runs in one process on one card, whose name, power
limit and SM clock are printed beside the numbers; without a GPU the script fails.

  pictures/s  4K, 16 distinct desktop frames as (3, H, W) tensors in [0, 1], the settings of bench.py's `value` leg (CBR
              20 Mbit/s, 60 fps, 64-picture steps, device-timed), --runs alternating fresh-session runs of each entry:
                idiom     (x.clamp(0, 1) * 255).round().to(torch.uint8).permute(1, 2, 0).contiguous() on torch's current
                          stream, then b2v_submit_device("RGB").  What users write; in fp16 it multiplies and rounds in fp16,
                          so its pixels can differ from the rule by one level: a timing comparator, not a parity one
                tensor    b2v_submit_tensor of the tensor as it is
                resident  b2v_submit_resident of the library's own BGRA copies: the ceiling
              for fp16, fp32 and uint8 (where the idiom is the transposing copy alone).
  csc         ms per CSC launch at 4K and 8K for planar tensors of each element type (B2V_FLAG_NO_ENCODE | B2V_FLAG_TIMING_CSC
              sessions: a CUDA-event pair around every 4th launch), as a fraction of 3.35 TB/s (H100 SXM data sheet) for the
              bytes the shapes give: 3 elements read and 1.5 B of NV12 written per pixel.
  general     the same at 4K for interleaved (H, W, 3) fp16 and for a planar fp16 window 3 pixels and 1 row into a larger
              surface (not 16-byte aligned): the general kernel.

Usage: python tools/tensor_ingest.py [--device 0] [--steps 16] [--warmup 2] [--runs 5] [--out FILE.json]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.device_ingest import FPS, H, HBM_GBS, KBPS, N_DISTINCT, STEP, W, card      # noqa: E402

ELEM = {"u8": 1, "f16": 2, "bf16": 2, "f32": 4}


def bytes_per_px(dtype: str) -> float:
    return 3 * ELEM[dtype] + 1.5


def throughput(submit, device: int, steps: int, warmup: int, resident=None) -> float:
    """Pictures/s of one fresh session fed by submit(session, k)."""
    from selkies_b200 import _native as N
    from selkies_b200.session import Session
    with Session(W, H, fps=FPS, device=device, rc_mode=N.B2V_RC_CBR, bitrate_kbps=KBPS, ring_slots=N_DISTINCT, collect=False) as s:
        for i, f in enumerate(resident or []):
            s.resident_upload(i, f)
        k = 0
        for _ in range(warmup * STEP):
            submit(s, k); k += 1
        s.flush()
        s.timer_start()
        for _ in range(steps * STEP):
            submit(s, k); k += 1
        ms = s.timer_stop()
    return steps * STEP / (ms / 1000.0)


def csc_ms(w, h, tensors, device: int, layout="CHW", origin=(0, 0), pictures: int = 512) -> float:
    """Mean ms per CSC launch (CUDA events around every 4th launch) of tensor submits."""
    from selkies_b200 import _native as N
    from selkies_b200.session import Session
    with Session(w, h, device=device, flags=N.B2V_FLAG_NO_ENCODE | N.B2V_FLAG_TIMING_CSC, ring_slots=8, collect=False) as s:
        for k in range(64):
            s.submit_tensor(tensors[k % len(tensors)], layout=layout, origin=origin)
        s.flush()
        s.reset_stats()
        for k in range(pictures):
            s.submit_tensor(tensors[k % len(tensors)], layout=layout, origin=origin)
        s.flush()
        st = s.stats()
    return st["ms_csc"] / max(1, st["n_csc"])


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
    from tests.tensor_scenario import device_tensor, host_tensor
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    dev = a.device
    torch.cuda.set_device(dev)
    res = {"card": card(dev)}
    print("card:", res["card"], flush=True)

    frames = [synth.desktop(W, H, t) for t in range(N_DISTINCT)]

    def idiom(x):
        if x.dtype == torch.uint8:
            return x.permute(1, 2, 0).contiguous()
        return (x.clamp(0, 1) * 255).round().to(torch.uint8).permute(1, 2, 0).contiguous()

    res["pictures_per_s"] = {}
    for dtype in ("f16", "f32", "u8"):
        tensors = [device_tensor(host_tensor(f, dtype)[0], device=dev)[0] for f in frames]
        entries = {
            "idiom": (lambda s, k: s.submit_device(idiom(tensors[k % N_DISTINCT]), pixel_format="RGB"), None),
            "tensor": (lambda s, k: s.submit_tensor(tensors[k % N_DISTINCT]), None),
            "resident": (lambda s, k: s.submit_resident(k % N_DISTINCT), frames),
        }
        runs = {k: [] for k in entries}
        for _ in range(a.runs):
            for name, (submit, resident) in entries.items():
                runs[name].append(throughput(submit, dev, a.steps, a.warmup, resident))
        res["pictures_per_s"][dtype] = {k: {"runs": [round(v, 1) for v in r], "min": round(min(r), 1), "max": round(max(r), 1)} for k, r in runs.items()}
        print(f"4K pictures/s, {dtype}:", json.dumps(res["pictures_per_s"][dtype]), flush=True)
        del tensors, entries
        torch.cuda.empty_cache()

    def frac(w, h, bpp, ms):
        return round(w * h * bpp / (ms * 1e-3) / 1e9 / HBM_GBS, 3)

    res["csc"] = []
    sizes = {"4K": (W, H, frames[:8]), "8K": (2 * W, 2 * H, [np.tile(f, (2, 2, 1)) for f in frames[:4]])}
    for name, (w, h, fr) in sizes.items():
        row = {"size": name}
        for dtype in ELEM:
            hosts = [host_tensor(f, dtype)[0] for f in fr]
            ms = csc_ms(w, h, [device_tensor(t, device=dev)[0] for t in hosts], dev)
            row[dtype] = {"bytes_per_px": bytes_per_px(dtype), "ms": round(ms, 4), "frac": frac(w, h, bytes_per_px(dtype), ms)}
            if name == "4K" and dtype == "f16":
                ms = csc_ms(w, h, [device_tensor(t, "HWC", device=dev)[0] for t in hosts], dev, layout="HWC")
                row["f16_interleaved"] = {"ms": round(ms, 4), "frac": frac(w, h, bytes_per_px(dtype), ms)}
                ms = csc_ms(w, h, [device_tensor(t, margin=(3, 1), device=dev)[0] for t in hosts], dev, origin=(3, 1))
                row["f16_unaligned_window"] = {"ms": round(ms, 4), "frac": frac(w, h, bytes_per_px(dtype), ms)}
            del hosts
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
