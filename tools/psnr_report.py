"""PSNR / SSIM / bitrate table of the CUDA encoder (SURVEY.md §8c.4 iii: decoded-vs-source quality per config and bitrate).
Every picture is measured on the GPU by the session itself (Session(quality=True), B2V_FLAG_QUALITY): the reconstruction, which
is what a decoder outputs, against the picture the encoder coded.
Run on the GPU box:  python tools/psnr_report.py  -> gpurun_out/psnr_report.json
The x264 comparator is absent from this image (probed at run time), so the table is absolute."""
import json, os, shutil, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import synth


def content(name, w, h, n):
    if name == "desktop_scroll":
        return [synth.desktop(w, h, t) for t in range(n)]
    if name == "bench_cycle16":               # bench.py's workload: 16 distinct pictures cycled (the scroll restarts every 16 pictures)
        fr = [synth.desktop(w, h, t) for t in range(16)]
        return [fr[t % 16] for t in range(n)]
    if name == "bars_box":
        return [synth.bars(w, h, t) for t in range(n)]
    if name == "gradient_pan":
        return [synth.gradient(w, h, t) for t in range(n)]
    if name == "static_desktop":
        f = synth.desktop(w, h, 0)
        return [f] * n
    raise ValueError(name)


_cache = {}


def prepared(w, h, name, n):
    """frames (made once per content and reused for every bitrate)."""
    key = (w, h, name, n)
    if key not in _cache:
        _cache.clear()
        _cache[key] = content(name, w, h, n)
    return _cache[key]


def run(w, h, name, kbps, fps, n):
    frames = prepared(w, h, name, n)
    with Session(w, h, fps=fps, rc_mode=N.B2V_RC_CBR, bitrate_kbps=kbps, ring_slots=4, quality=True) as s:
        for f in frames:
            s.submit(f)
        s.flush()
        got = s.take_frames()
    assert len(got) == n
    tail = range(n // 2, n)              # steady state: the second half, after the key-frame burst has been absorbed
    ps = {i: got[i].quality.psnr for i in range(n)}
    sizes = [len(g.data) for g in got]
    tl = [i for i in tail if i != 0] or [0]
    win = int(fps)
    tb = kbps * 1000.0 / fps / 8.0             # target bytes per picture
    windows = [sum(sizes[i:i + win]) / (tb * win) for i in range(0, max(1, n - win + 1))]
    qps = [g.qp for g in got]
    return {"w": w, "h": h, "content": name, "target_kbps": kbps, "fps": fps, "frames": n,
            "achieved_kbps_steady": float(np.mean([sizes[i] for i in tail]) * 8 * fps / 1000),
            "achieved_over_target_steady": float(np.mean([sizes[i] for i in tail]) / tb),
            "worst_1s_window_over_target": float(max(windows)), "worst_1s_window_after_the_first_second": float(max(windows[win:])) if len(windows) > win else None,
            "qp_pinned": "max" if min(qps[n // 2:]) >= 51 else "min" if max(qps[n // 2:]) <= 10 else None, "idr_bytes": sizes[0],
            "psnr_y_steady": float(np.mean([ps[i][0] for i in tl])), "psnr_u_steady": float(np.mean([ps[i][1] for i in tl])),
            "psnr_v_steady": float(np.mean([ps[i][2] for i in tl])), "psnr_y_idr": ps[0][0],
            "ssim_y_steady": float(np.mean([got[i].quality.ssim for i in tl])), "ssim_y_idr": got[0].quality.ssim,
            "psnr_y_min": float(min(ps[i][0] for i in range(n))),
            "qp_first_last": [got[0].qp, got[-1].qp], "qp_steady_mean": float(np.mean([got[i].qp for i in tail]))}


def main():
    os.makedirs("gpurun_out", exist_ok=True)
    rows = []
    for (w, h) in [(1920, 1080), (3840, 2160)]:
        for name in ["desktop_scroll", "bench_cycle16", "bars_box", "gradient_pan", "static_desktop"]:
            for kbps in [8000, 20000, 50000, 100000]:
                r = run(w, h, name, kbps, 60.0, 240 if w == 1920 else 180)
                rows.append(r)
                print(json.dumps(r), flush=True)
    out = {"x264_comparator": shutil.which("x264") or "absent", "gst_launch": shutil.which("gst-launch-1.0") or "absent",
           "rate_control": "CBR (settings.py:49 range 1-100 Mbps); bucket + ratio controller, QP 10..51, feedback two pictures late (DESIGN.md 5.6)",
           "reading": "achieved_over_target_steady is over the second half of the run; qp_pinned = the controller sat at its limit there (content cannot use / cannot fit the budget)",
           "rows": rows}
    json.dump(out, open("gpurun_out/psnr_report.json", "w"), indent=1)


if __name__ == "__main__":
    main()
