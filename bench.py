#!/usr/bin/env python
"""bench.py — headline benchmark of the H100-native video hot path (see DESIGN.md §7).

Workload (BASELINE.json metric "4K frames/sec encoded per GPU", configs[2]): synthetic desktop-like
3840x2160 BGRA frames -> fused BT.709 CSC -> H.264 Constrained-Baseline (one IDR, then P pictures with
the exhaustive warp-SAD motion search), CBR 20 Mbit/s @ 60 fps nominal, free-running.
A STEP is one batch of FRAMES_PER_STEP frames through one session (one session per GPU).

  value  frames/s with the BGRA inputs already resident in HBM (b2v_submit_resident), device-timed
  e2e    frames/s through the host-buffer API: pinned host ring -> cudaMemcpyAsync H2D -> CSC -> encode
         -> D2H of every access unit -> Python callback, wall-clock + device timer inside the timed region
  roofline       the fused CSC kernel: algorithmic bytes (5.5 B/px) / CUDA-event time per launch, in-step, as a fraction of
                 the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s)
  cpu_baseline   the CPU restatement (oracle/) on the host cores, bounded sample (rank 0, N=1 only)

`--impl reference` times the CPU path only (the reference's own videoconvert+x264enc pipeline cannot
run here — SURVEY.md §8c — so the arm runs the oracle port, all host threads, labelled kind="port").

`--dump-outputs DIR` writes what the timed leg delivered in its last step — the access units of its FRAMES_PER_STEP pictures —
as DIR/*.npy (float32 / float64), so that two builds can be compared output for output on identical inputs.  Capturing them
needs a Python callback on the timed session, which slows and spreads `value`: take timings from a run without it.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

W, H = 3840, 2160
FPS_NOMINAL = 60.0
BITRATE_KBPS = 20000
FRAMES_PER_STEP = 64      # one step = one batch of 64 pictures through the hot path (long enough that host scheduling jitter averages out)
N_DISTINCT = 16           # distinct input frames cycled (the scroll restarts every 16 pictures): 16 x 33.2 MB = 531 MB > 50 MB of L2
N_SIDE = 256              # pictures in each side measurement (device-timer pass, striped mode)
ALG_BYTES_PER_PX = 5.5    # 4 B BGRA read + 1 B Y + 0.5 B CbCr written (SURVEY.md §8d)
HBM_PEAK_GBS = 3350.0     # H100 SXM data sheet (HBM3, 700 W card); a roofline fraction is achieved / this, never a measured peak
DUMP_MAX_BYTES = 16 << 20 # --dump-outputs: at most 16 Mi access-unit bytes (64 MB as float32); more is sampled with a fixed seed


def synth_frames(n, w=W, h=H):
    from tests import synth
    return [synth.desktop(w, h, t) for t in range(n)]


class ClockSampler:
    """nvidia-smi clocks + throttle reasons DURING the timed region.  One nvidia-smi process
    (rank 0 only, all GPUs of the job, 100 ms period) is started before the warm-up so that it is already streaming when the
    timed region begins; `mark()` / `stop()` delimit the rows that fall inside it."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, n_gpus: int):
        self.n_gpus, self.rows, self.proc, self.t_mark = n_gpus, [], None, None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.monotonic(), [c.strip() for c in line.split(",")]))

    def mark(self):
        self.t_mark = time.monotonic()

    def stop(self):
        t_end = time.monotonic()
        if self.proc:
            time.sleep(0.11)                 # let the sample that was being taken at t_end arrive
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except Exception:
                pass
        mine = [(t, r) for t, r in self.rows if len(r) >= 8 and r[0].isdigit() and int(r[0]) < self.n_gpus]
        inside = [r for t, r in mine if self.t_mark is not None and self.t_mark <= t <= t_end + 0.11]
        window = "timed region"
        if not inside and mine:              # region shorter than one sampling period: the samples bracketing it
            t0 = self.t_mark if self.t_mark is not None else t_end
            near = sorted(mine, key=lambda tr: min(abs(tr[0] - t0), abs(tr[0] - t_end)))[: 2 * self.n_gpus]
            inside, window = [r for _, r in near], "nearest samples (region shorter than the 100 ms period)"
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in inside:
            try:
                sm.append(float(r[1])); mx.append(float(r[2]))
                for n, v in zip(names, r[4:8]):
                    if v.lower().startswith("active"):
                        reasons.add(n)
            except Exception:
                pass
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        return {"sm_mhz": float(np.median(sm)), "sm_min_mhz": float(min(sm)), "sm_max_mhz": float(max(mx)), "reasons": sorted(reasons),
                "samples": len(sm), "window": window, "gpus_sampled": self.n_gpus}


def cpu_quota():
    """CPUs this container may actually use (cgroup v2 cpu.max), or None when unlimited/unknown."""
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()
        return None if q == "max" else float(q) / float(p)
    except Exception:
        return None


def bind_to_gpu_numa_node(torch, device: int):
    """Best effort: restrict this rank to the CPUs of the NUMA node its GPU hangs off, BEFORE the pinned host ring is
    allocated (first-touch placement), so that 8 concurrent sessions do not all pull their 33 MB frames across sockets."""
    try:
        pr = torch.cuda.get_device_properties(device)
        bdf = f"{pr.pci_domain_id:04x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0"
        node = int(open(f"/sys/bus/pci/devices/{bdf}/numa_node").read())
        if node < 0:
            return None
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
        allowed = cpus & os.sched_getaffinity(0)
        if allowed:
            os.sched_setaffinity(0, allowed)
        return node
    except Exception:
        return None


def usable_threads() -> int:
    """All the host threads the container may really use: min(online CPUs, cgroup quota rounded up)."""
    n = os.cpu_count() or 1
    q = cpu_quota()
    return max(1, min(n, int(q + 0.999))) if q else n


def cpu_sample(frames, n_p: int, threads: int | None = None, keep=None):
    """Oracle CSC + encode of 1 IDR + n_p P pictures on the host cores; returns (P frames/s, seconds, threads).  `keep`: a list
    that receives the access units (the checker's output, compared with the GPU's by parity_leg)."""
    import oracle
    used = oracle.set_threads(threads or usable_threads())
    enc = oracle.RefEncoder(W, H)
    target = int(BITRATE_KBPS * 1000 / FPS_NOMINAL)
    au = enc.encode_bgra(frames[0], True, rc_mode=0, target_bits=target)
    if keep is not None:
        keep.append(au)
    t0 = time.perf_counter()
    for i in range(n_p):
        au = enc.encode_bgra(frames[(i + 1) % len(frames)], False, rc_mode=0, target_bits=target)
        if keep is not None:
            keep.append(au)
    dt = time.perf_counter() - t0
    return n_p / dt, dt, used


def x264_anchor(cores: int):
    """The only published number for the reference's own CPU encoder: docs/design.md:33 — 1080p60 costs about 1.5 cores of
    x264enc (ultrafast/zerolatency) + videoconvert.  Scaled by pixel count (4K = 4 x 1080p) that is ~6 cores for 4K60, i.e.
    ~10 pictures/s per core; on `cores` host cores ~10*cores pictures/s.  An ESTIMATE from a published anchor on other
    hardware, not a measurement: x264 / GStreamer are absent from this image (SURVEY.md §8c)."""
    per_core = 60.0 / (1.5 * 4.0)
    return {"frames_per_s_estimate": per_core * cores, "cores": cores, "per_core": per_core,
            "source": "reference docs/design.md:33 (1080p60 ~ 150 % CPU), scaled x4 pixels; estimate, not measured here"}


def run_reference(args, rank, world):
    """CPU arm: the oracle port on all host threads; a step = 1 P picture of the same workload."""
    if rank != 0:
        return
    frames = synth_frames(N_DISTINCT)          # the same cycle of pictures as the GPU arm
    import oracle
    cores = oracle.set_threads(usable_threads())
    enc = oracle.RefEncoder(W, H)
    target = int(BITRATE_KBPS * 1000 / FPS_NOMINAL)
    enc.encode_bgra(frames[0], True, rc_mode=0, target_bits=target)
    for i in range(args.warmup):
        enc.encode_bgra(frames[(i + 1) % len(frames)], False, rc_mode=0, target_bits=target)
    t0 = time.perf_counter()
    for i in range(args.steps):
        enc.encode_bgra(frames[(i + 1 + args.warmup) % len(frames)], False, rc_mode=0, target_bits=target)
    dt = time.perf_counter() - t0
    fps = args.steps / dt
    line = {
        "impl": "reference", "metric": "4K frames/sec encoded", "value": fps, "unit": "frames/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1000 * dt / args.steps, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": workload_config(1),
        "cpu_baseline": {"value": fps, "unit": "frames/s", "cores": cores, "cgroup_cpu_quota": cpu_quota(), "kind": "port",
                         "sample": f"{args.steps} P pictures 3840x2160 (CSC + encode), OpenMP over macroblock rows; "
                                   "the reference's videoconvert+x264enc is absent from this image"},
        "e2e": {"value": fps, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    emit(line)


def rtp_leg(aus):
    """SURVEY.md §8f row 1: native RTP H.264 payloader vs the Python restatement of the reference's (host code)."""
    if not aus:
        return None
    try:
        from oracle import rtp_ref
        from selkies_b200.rtp_h264 import H264Payloader
        pl = H264Payloader()
        reps = 20
        t0 = time.perf_counter()
        for _ in range(reps):
            for au in aus:
                n = len(pl.packetize(au))
        t_native = (time.perf_counter() - t0) / (reps * len(aus))
        t0 = time.perf_counter()
        for au in aus:
            ref = rtp_ref.pack_access_unit(au)
        t_py = (time.perf_counter() - t0) / len(aus)
        same = all(pl.packetize(au) == rtp_ref.pack_access_unit(au) for au in aus)
        return {"au_bytes": sum(map(len, aus)) / len(aus), "packets_per_au": len(ref), "native_us_per_au": t_native * 1e6,
                "python_reference_port_us_per_au": t_py * 1e6, "identical_payloads": same}
    except Exception as e:
        return {"error": repr(e)}


HOST_KEYS = ("ns_wait_event", "ns_wait_job", "ns_callback", "ns_wait_out_slot", "ns_wait_ring", "ns_submit")


def host_breakdown(st1, st0, n_frames):
    """Where this session's HOST threads spent the leg, in microseconds per picture (b2v_stats stopwatches): the output thread
    waiting for the GPU / idle / inside the callback, the submitter blocked on back-pressure or inside CUDA enqueue calls."""
    d = {k[3:] + "_us": (st1[k] - (st0[k] if st0 else 0)) / 1e3 / max(1, n_frames) for k in HOST_KEYS}
    d["wait_event_max_us"] = st1["ns_wait_event_max"] / 1e3
    d["event_sleeps_per_frame"] = (st1["n_event_sleeps"] - (st0["n_event_sleeps"] if st0 else 0)) / max(1, n_frames)
    return d


def resident_leg(frames, n_pics, device, *, w=W, h=H, warm=32, collect_sizes=False, **kw):
    """Side measurement: `n_pics` pictures of `frames` (cycled, resident in HBM) through a fresh session, device-timed."""
    from selkies_b200.session import Session
    nb = [0, 0]

    def on_frame(fptr):
        nb[0] += fptr.contents.size; nb[1] += 1
    with Session(w, h, device=device, collect=False, on_frame=on_frame, **kw) as ss:
        for i, f in enumerate(frames):
            ss.resident_upload(i, f)
        for k in range(warm):
            ss.submit_resident(k % len(frames))
        ss.flush(); nb[0] = nb[1] = 0
        ss.timer_start()
        for k in range(n_pics):
            ss.submit_resident((warm + k) % len(frames))
        ms = ss.timer_stop()
    return {"value": n_pics / (ms / 1000.0), "unit": "frames/s", "ms_per_picture": ms / n_pics, "pictures": n_pics,
            "bytes_per_picture": nb[0] / max(1, n_pics), "callbacks_per_picture": nb[1] / max(1, n_pics)}


def parity_leg(frames, ref_aus, device):
    """The first len(ref_aus) access units of the bench stream (fresh session, same settings and entry point as the timed leg)
    compared byte for byte with the checker's (oracle) output for the same pictures."""
    from selkies_b200 import _native as N
    from selkies_b200.session import Session
    with Session(W, H, fps=FPS_NOMINAL, device=device, rc_mode=N.B2V_RC_CBR, bitrate_kbps=BITRATE_KBPS, ring_slots=N_DISTINCT,
                 flags=N.B2V_FLAG_TIMING_CSC) as sp:
        for i, f in enumerate(frames):
            sp.resident_upload(i, f)
        for i in range(len(ref_aus)):
            sp.submit_resident(i % len(frames))
        sp.flush()
        got = sp.take_frames()
    bad = [i for i, (g, r) in enumerate(zip(got, ref_aus)) if g.data != r]
    return {"parity_checked": len(ref_aus), "parity_ok": not bad and len(got) == len(ref_aus), "first_mismatch": bad[0] if bad else None,
            "what": "access-unit bytes, GPU vs oracle, 1 IDR + P pictures of the timed workload (incl. the scroll restart at picture 16)"}


def python_surface_leg(frames, device, seconds=2.0):
    """SURVEY §7 / VERDICT r1 Missing #8: 4K throughput through the reference-facing PYTHON surface — pixelflux_compat.ScreenCapture
    fed by an ArraySource (a numpy copy of every 33 MB frame into the pinned slot, the job of the reference's XShm grab), the
    callback doing what media_pipeline.py:286 does: bytes(result.data[10:result.size])."""
    from selkies_b200.pixelflux_compat import ArraySource, CaptureSettings, ScreenCapture
    n, nbytes = [0], [0]

    def cb(result_ptr, _user):
        if not result_ptr:
            return
        r = result_ptr.contents
        au = bytes(r.data[10:r.size])
        n[0] += 1; nbytes[0] += len(au)
    cs = CaptureSettings()
    cs.capture_width, cs.capture_height, cs.target_fps = W, H, 1000.0       # free-running: the source never has to wait
    cs.h264_cbr_mode, cs.h264_bitrate_kbps, cs.gpu_id = True, BITRATE_KBPS, device
    cap = ScreenCapture(ArraySource(frames, loop=True))
    cap.start_capture(cs, cb)
    time.sleep(0.5)
    n0, t0 = n[0], time.perf_counter()
    time.sleep(seconds)
    n1, t1 = n[0], time.perf_counter()
    cap.stop_capture()
    return {"value": (n1 - n0) / (t1 - t0), "unit": "frames/s", "seconds": t1 - t0,
            "note": "ScreenCapture + ArraySource(4K) -> callback bytes(result.data[10:size]); includes the producer's 33 MB numpy copy "
                    "into the pinned slot per frame (single Python thread), H2D, encode, D2H"}


def dump_outputs(out_dir, aus):
    """The access units a caller of the timed path received in its last step: their bytes concatenated (float32; a seeded sample
    when longer than DUMP_MAX_BYTES), and per picture the size, QP and key-frame flag (float64)."""
    if len(aus) != FRAMES_PER_STEP:
        raise RuntimeError(f"--dump-outputs: {len(aus)} access units captured from the last step, expected {FRAMES_PER_STEP}")
    os.makedirs(out_dir, exist_ok=True)
    data = np.frombuffer(b"".join(a for a, _, _ in aus), np.uint8)
    if data.size > DUMP_MAX_BYTES:
        data = data[np.sort(np.random.default_rng(0).choice(data.size, DUMP_MAX_BYTES, replace=False))]
    np.save(os.path.join(out_dir, "access_unit_bytes.npy"), data.astype(np.float32))
    np.save(os.path.join(out_dir, "access_unit_sizes.npy"), np.array([len(a) for a, _, _ in aus], np.float64))
    np.save(os.path.join(out_dir, "access_unit_qp.npy"), np.array([q for _, _, q in aus], np.float64))
    np.save(os.path.join(out_dir, "access_unit_is_key.npy"), np.array([k for _, k, _ in aus], np.float64))


def workload_config(frames_per_step):
    return {"workload": "C2: 3840x2160 synthetic desktop BGRA -> fused BT.709 CSC -> H.264 CBP (IDR then P; full-sample ME +-16: zero / temporal / anchor predictors in front of an exhaustive search, quarter-sample refinement; Intra4x4/16x16 in IDR; CAVLC)",
            "frames_per_step": frames_per_step, "rate_control": f"CBR {BITRATE_KBPS} kbit/s @ {FPS_NOMINAL:g} fps nominal, free-running",
            "slice_rows": "default (P pictures: 8 macroblock rows per slice, IDR pictures: sub-row slices)", "sessions_per_gpu": 1,
            "l2_policy": f"inputs larger than L2: {N_DISTINCT} distinct frames x 33.2 MB cycled", "parallelism": "one independent session per GPU (no collective)"}


_REAL_STDOUT = None


def own_stdout():
    """stdout carries exactly ONE line (the JSON result): everything else that writes to fd 1 — NCCL's version banner, library
    chatter of any rank — is sent to stderr from here on."""
    global _REAL_STDOUT
    if _REAL_STDOUT is None:
        sys.stdout.flush()
        _REAL_STDOUT = os.dup(1)
        os.dup2(2, 1)


def emit(line: dict):
    data = (json.dumps(line) + "\n").encode()
    os.write(_REAL_STDOUT if _REAL_STDOUT is not None else 1, data)


def main():
    own_stdout()
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the access units of the last timed step to DIR/*.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if args.warmup < 3:
        args.warmup = 3
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))

    if args.impl == "reference":
        run_reference(args, rank, world)
        return

    import torch
    import torch.distributed as dist
    from selkies_b200 import _native as N
    from selkies_b200.session import Session

    torch.cuda.set_device(local_rank)
    numa = bind_to_gpu_numa_node(torch, local_rank)      # pinned ring + output buffers land next to this GPU's PCIe root
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(x: float) -> float:
        if world == 1:
            return x
        t = torch.tensor([x], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def gather_over_ranks(x: float):
        if world == 1:
            return [x]
        t = torch.zeros(world, dtype=torch.float64, device="cuda")
        t[rank] = x
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return [float(v) for v in t.tolist()]

    from selkies_b200.multi_gpu import aggregate_throughput, gather_over_ranks as gather_ranks, session_device
    assert world == 1 or session_device(rank, world) == local_rank       # one session per GPU, session i on GPU i mod n (SURVEY.md §8e)

    def gather_dict(d: dict):
        return gather_ranks(d, device="cuda")

    def sum_over_ranks(x: float) -> float:
        if world == 1:
            return x
        t = torch.tensor([x], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return float(t.item())

    frames = synth_frames(N_DISTINCT)
    peak, peak_src = HBM_PEAK_GBS, "H100 SXM data sheet, HBM3 3.35 TB/s"
    # leg 1 (`value`, inputs resident) and leg 2 (`e2e`) run with no instrumentation; the CUDA-event pairs around the CSC launches
    # that `roofline` is computed from sit in leg 1b: the same resident-input steps, timed the same way, with
    # B2V_FLAG_TIMING_CSC on (an event pair around the CSC launch of every 4th picture).  The events cost a GPU-bound step 4-5 %,
    # which is why `value` is not quoted from that leg; in the PCIe-bound e2e leg the GPU idles between pictures and an event
    # pair there mostly measures wake-up latency (29 us around a 9 us kernel)
    # leg 1 registers no Python callback: a per-picture callback has to take the GIL from the submitting thread on every picture,
    # and that hand-off, not the GPU, then sets the pace and the run-to-run spread.  Its byte counts come from the session's
    # stats.  Only --dump-outputs adds a callback, which copies the access units of the last timed step.
    # The session delivers one access unit per picture, in order; the pictures of the last timed step are delivered pictures
    # [first, first + FRAMES_PER_STEP) counted from the session's start.
    n_delivered = [0]
    dump_first = (args.warmup + args.steps - 1) * FRAMES_PER_STEP
    dump_aus = []

    def capture_last_step(fptr):
        if dump_first <= n_delivered[0] < dump_first + FRAMES_PER_STEP:
            f = fptr.contents
            dump_aus.append((ctypes.string_at(f.data, f.size), f.is_key, f.qp))
        n_delivered[0] += 1
    sess = Session(W, H, fps=FPS_NOMINAL, device=local_rank, rc_mode=N.B2V_RC_CBR, bitrate_kbps=BITRATE_KBPS,
                   ring_slots=N_DISTINCT, flags=0, collect=False, on_frame=capture_last_step if args.dump_outputs else None)

    # ---------------- leg 1: inputs resident in HBM ----------------------------------------------------
    for i, f in enumerate(frames):
        sess.resident_upload(i, f)

    def step_resident(k0):
        for j in range(FRAMES_PER_STEP):
            sess.submit_resident((k0 + j) % N_DISTINCT)

    clocks = ClockSampler(world) if rank == 0 else None
    if clocks:
        clocks.start()
    k = 0
    for _ in range(args.warmup):
        step_resident(k); k += FRAMES_PER_STEP
    sess.flush()
    sess.reset_stats()
    import gc
    gc.disable()                 # no collector pauses inside the timed regions
    barrier()
    if clocks:
        clocks.mark()
    sess.timer_start()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step_resident(k); k += FRAMES_PER_STEP
    dev_ms = sess.timer_stop()
    wall_ms = 1000 * (time.perf_counter() - t0)
    barrier()
    st = sess.stats()
    n_frames = args.steps * FRAMES_PER_STEP
    value, t_ms = aggregate_throughput(float(n_frames), max(dev_ms, 1e-6), device="cuda")      # sum of pictures / max time over ranks
    per_rank_ms = gather_over_ranks(max(dev_ms, 0.0))
    per_rank_wall_ms = gather_over_ranks(wall_ms)
    host_resident = gather_dict(host_breakdown(st, None, n_frames))       # reset_stats ran right before the leg

    # ---------------- leg 1b: the same steps with the CSC event pairs on (roofline) ----------------------------------
    with Session(W, H, fps=FPS_NOMINAL, device=local_rank, rc_mode=N.B2V_RC_CBR, bitrate_kbps=BITRATE_KBPS,
                 ring_slots=N_DISTINCT, flags=N.B2V_FLAG_TIMING_CSC, collect=False) as sr:
        for i, f in enumerate(frames):
            sr.resident_upload(i, f)
        kk = 0
        for _ in range(args.warmup):
            for j in range(FRAMES_PER_STEP):
                sr.submit_resident((kk + j) % N_DISTINCT)
            kk += FRAMES_PER_STEP
        sr.flush(); sr.reset_stats()
        barrier()
        sr.timer_start()
        for _ in range(args.steps):
            for j in range(FRAMES_PER_STEP):
                sr.submit_resident((kk + j) % N_DISTINCT)
            kk += FRAMES_PER_STEP
        roof_ms = sr.timer_stop()
        barrier()
        st_roof = sr.stats()

    # ---------------- leg 2: end to end from pinned host buffers -----------------------------------------
    # pre-fill the pinned ring once (the producer — XShm grab in the reference — writes into these slots);
    # every frame is then copied H2D inside the timed region and every access unit copied back D2H to a Python callback.
    out_bytes = [0]
    sample_aus = []

    def on_frame(fptr):
        out_bytes[0] += fptr.contents.size
        if len(sample_aus) < 8 and not fptr.contents.is_key:
            sample_aus.append(ctypes.string_at(fptr.contents.data, fptr.contents.size))
    se = Session(W, H, fps=FPS_NOMINAL, device=local_rank, rc_mode=N.B2V_RC_CBR, bitrate_kbps=BITRATE_KBPS,
                 ring_slots=N_DISTINCT, flags=0, collect=False, on_frame=on_frame)
    for i in range(N_DISTINCT):
        slot, view = se.acquire()
        view[...] = frames[i]
        se.submit_slot(slot)
    se.flush()

    def step_host():
        for _ in range(FRAMES_PER_STEP):
            slot, _view = se.acquire()       # round-robin: slot i still holds distinct frame i
            se.submit_slot(slot)

    for _ in range(args.warmup):
        step_host()
    se.flush()
    st0 = se.stats()
    out_bytes[0] = 0
    barrier()
    se.timer_start()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step_host()
    e2e_dev_ms = se.timer_stop()
    e2e_wall_ms = 1000 * (time.perf_counter() - t0)
    barrier()
    clk = clocks.stop() if clocks else None
    st1 = se.stats()
    se.close()
    e2e_ms = max_over_ranks(max(e2e_wall_ms, e2e_dev_ms))
    e2e_value = sum_over_ranks(float(n_frames)) / (e2e_ms / 1000.0)
    per_rank_e2e_ms = gather_over_ranks(max(e2e_wall_ms, e2e_dev_ms))
    host_e2e = gather_dict(host_breakdown(st1, st0, n_frames))
    h2d_step = (st1["h2d_bytes"] - st0["h2d_bytes"]) / args.steps
    d2h_step = (st1["d2h_bytes"] - st0["d2h_bytes"]) / args.steps

    # ---------------- roofline of the fused CSC kernel (in-step CUDA-event pairs) -------------------------
    alg = W * H * ALG_BYTES_PER_PX
    csc_ms = st_roof["ms_csc"] / max(1, st_roof["n_csc"])       # event pairs of the instrumented resident leg (1b)
    achieved = alg / (csc_ms * 1e-3) / 1e9 if csc_ms > 0 else 0.0
    burst_ms = sess.bench_csc_burst(N_DISTINCT, 200)
    roofline = {"bound": "hbm", "kernel": "csc_bgra_nv12_fast", "achieved": achieved, "peak": peak, "unit": "GB/s",
                "frac": achieved / peak, "peak_source": peak_src,
                "algorithmic_bytes_per_launch": alg, "us_per_launch": csc_ms * 1e3,
                "timed_launches": int(st_roof["n_csc"]),
                "where": "CUDA-event pair around the CSC launch of every 4th picture of leg 1b: the resident-input steps of `value`, re-run with the events on "
                         f"({n_frames / (roof_ms / 1000.0):.0f} frames/s with them)",
                "device_timer": None,
                "burst": {"note": f"200 back-to-back launches between one event pair, same {N_DISTINCT} cycled frames",
                          "us_per_launch": burst_ms * 1e3, "achieved": alg / (burst_ms * 1e-3) / 1e9,
                          "frac": alg / (burst_ms * 1e-3) / 1e9 / peak}}
    # the same step with the CSC kernel stamping %globaltimer itself (first block start .. last block end): shows what the
    # event pair adds (two event commands + the launch gap around an 8-9 us kernel).  Separate short pass: the stamps cost two
    # memsets and two atomics per block, which must not perturb the timed region above.
    if rank == 0:
        try:
            with Session(W, H, fps=FPS_NOMINAL, device=local_rank, rc_mode=N.B2V_RC_CBR, bitrate_kbps=BITRATE_KBPS, ring_slots=4,
                         flags=N.B2V_FLAG_TIMING | N.B2V_FLAG_DEVICE_TIMER, collect=False) as sd:
                for i, f in enumerate(frames):
                    sd.resident_upload(i, f)
                for kk in range(48):
                    sd.submit_resident(kk % N_DISTINCT)
                sd.flush(); sd.reset_stats()
                for kk in range(N_SIDE):
                    sd.submit_resident(kk % N_DISTINCT)
                sd.flush()
                sdt = sd.stats()
            if sdt["n_csc_device"]:
                us = sdt["ms_csc_device"] / sdt["n_csc_device"] * 1e3
                roofline["device_timer"] = {"note": "in-step launches timed by the kernel itself (%globaltimer), 256 pictures, separate instrumented pass",
                                            "us_per_launch": us, "achieved": alg / (us * 1e-6) / 1e9, "frac": alg / (us * 1e-6) / 1e9 / peak}
        except Exception as e:
            roofline["device_timer"] = {"error": repr(e)}
    # per-kernel breakdown: separate pass with every stage bracketed by events (those extra event commands cost the step 4-5 %,
    # so they stay out of the timed legs)
    with Session(W, H, fps=FPS_NOMINAL, device=local_rank, rc_mode=N.B2V_RC_CBR, bitrate_kbps=BITRATE_KBPS, ring_slots=4,
                 flags=N.B2V_FLAG_TIMING, collect=False) as sk:
        for i, f in enumerate(frames):
            sk.resident_upload(i, f)
        for kk in range(48):
            sk.submit_resident(kk % N_DISTINCT)
        sk.flush(); sk.reset_stats()
        for kk in range(N_SIDE):
            sk.submit_resident(kk % N_DISTINCT)
        sk.flush()
        stk = sk.stats()
    kern = {k: (stk["ms_" + k] / max(1, stk["n_" + k])) * 1e3 for k in ("csc", "intra", "inter", "cavlc", "slice", "pack")}
    kern["gpu_span_per_frame"] = stk["ms_total_gpu"] / max(1, stk["n_csc"]) * 1e3
    kern["note"] = f"separate instrumented pass, {N_SIDE} pictures, every stage between CUDA events"
    per_rank_span = gather_over_ranks(kern["gpu_span_per_frame"])
    per_rank_inter = gather_over_ranks(kern["inter"])
    per_rank_numa = gather_over_ranks(float(-1 if numa is None else numa))
    sess.close()
    # BASELINE config 4 (7680x4320 CSC roofline stress): same kernel, one event pair per launch, 4 frames x 132.7 MB cycled
    if rank == 0:
        try:
            from tests import synth
            w8, h8 = 7680, 4320
            tile = synth.desktop(1920, 1080, 0)
            f8 = np.tile(tile, (4, 4, 1))
            with Session(w8, h8, device=local_rank, flags=N.B2V_FLAG_NO_ENCODE) as s8:
                for i in range(4):
                    s8.resident_upload(i, np.roll(f8, 16 * i, axis=1))
                ms8 = s8.bench_csc(4, 60)
                ms8b = s8.bench_csc_burst(4, 60)
            alg8 = w8 * h8 * ALG_BYTES_PER_PX
            roofline["c4_8k_stress"] = {"us_per_launch": ms8 * 1e3, "achieved": alg8 / (ms8 * 1e-3) / 1e9, "frac": alg8 / (ms8 * 1e-3) / 1e9 / peak,
                                        "burst_us_per_launch": ms8b * 1e3, "burst_frac": alg8 / (ms8b * 1e-3) / 1e9 / peak,
                                        "algorithmic_bytes_per_launch": alg8, "note": "one CUDA-event pair per launch; 4 resident frames cycled (531 MB > L2)"}
        except Exception as e:
            roofline["c4_8k_stress"] = {"error": repr(e)}

    # ---------------- fused scale + CSC legs (VERDICT r1 N1): 4K -> 1080p and 1080p -> 4K, same event-pair timing as the 1:1 kernel ----
    if rank == 0:
        try:
            from tests import synth
            sc = {}
            for (sw, sh, dw, dh) in ((3840, 2160, 1920, 1080), (1920, 1080, 3840, 2160)):
                with Session(sw, sh, dst_width=dw, dst_height=dh, device=local_rank, flags=N.B2V_FLAG_NO_ENCODE) as sx:
                    nres = 8 if sw > 2000 else 24
                    base = synth.desktop(sw, sh, 0)
                    for i in range(nres):
                        sx.resident_upload(i, np.roll(base, 8 * i, axis=0))
                    ms_e, ms_b = sx.bench_csc(nres, 100), sx.bench_csc_burst(nres, 100)
                algs = 4.0 * sw * sh + 1.5 * dw * dh
                sc[f"{sw}x{sh}_to_{dw}x{dh}"] = {"us_per_launch": ms_e * 1e3, "burst_us_per_launch": ms_b * 1e3, "algorithmic_bytes_per_launch": algs,
                                                 "achieved": algs / (ms_e * 1e-3) / 1e9, "frac": algs / (ms_e * 1e-3) / 1e9 / peak,
                                                 "burst_frac": algs / (ms_b * 1e-3) / 1e9 / peak}
            sc["note"] = "csc_bgra_nv12_scaled (shared-memory tile, bilinear + BT.709 in one pass); bytes = 4 B x source px + 1.5 B x output px; one CUDA-event pair per launch"
            roofline["scaled"] = sc
        except Exception as e:
            roofline["scaled"] = {"error": repr(e)}

    # ---------------- side legs (rank 0): striped mode, IDR / C1, worst-case contents, the Python surface ----------------
    striped = idr_legs = content_legs = py_surface = None
    if rank == 0:
        cbr = dict(fps=FPS_NOMINAL, rc_mode=N.B2V_RC_CBR, bitrate_kbps=BITRATE_KBPS, ring_slots=4)
        try:      # SURVEY.md §8f row 2: same frames, 8 independent stripes per picture
            rows = -(-(H // 16) // 8)
            striped = resident_leg(frames, N_SIDE, local_rank, warm=48, stripe_rows=rows, header_mode=N.B2V_HDR_PIXELFLUX, **cbr)
            striped.update({"stripe_rows": rows, "stripes_per_picture": -(-(H // 16) // rows),
                            "stripes_delivered_per_picture": striped.pop("callbacks_per_picture"),
                            "note": "inputs resident in HBM, 256 pictures; stripes whose macroblocks were all skipped are not delivered"})
        except Exception as e:
            striped = {"error": repr(e)}
        try:      # VERDICT r1 N2: the IDR path (PLI -> key frame, rtc.py:601-603) and BASELINE configs[1] (1080p60, I-only)
            from tests import synth
            i4k = resident_leg(frames, 48, local_rank, warm=8, gop=1, **cbr)
            i4q = resident_leg(frames, 48, local_rank, warm=8, gop=1, fps=FPS_NOMINAL, rc_mode=N.B2V_RC_CQP, crf=30, ring_slots=4)
            f1080 = [synth.desktop(1920, 1080, t) for t in range(N_DISTINCT)]
            c1 = resident_leg(f1080, 128, local_rank, w=1920, h=1080, warm=16, gop=1, fps=60.0, rc_mode=N.B2V_RC_CQP, crf=25, ring_slots=4)
            idr_legs = {"idr_4k_ms": i4k["ms_per_picture"], "i_only_4k_fps": i4k["value"], "idr_4k_bytes": i4k["bytes_per_picture"],
                        "idr_4k_qp30_ms": i4q["ms_per_picture"], "idr_4k_qp30_bytes": i4q["bytes_per_picture"],
                        "c1_1080p_i_only_fps": c1["value"], "c1_1080p_idr_ms": c1["ms_per_picture"], "c1_bytes_per_picture": c1["bytes_per_picture"],
                        "note": "gop=1 (every picture an IDR with in-band SPS/PPS), inputs resident; 4K: CBR 20 Mbit/s; C1 = BASELINE configs[1] "
                                "1920x1080 synthetic desktop, constant QP 25 (the reference's default h264_crf, settings.py:48), target 60 fps"}
        except Exception as e:
            idr_legs = {"error": repr(e)}
        try:      # worst-case contents: S2 uniform noise (nothing predictable, every MB searched + refined), S4 gradient pan
            from tests import synth
            s2 = resident_leg([synth.noise(W, H, 100 + t) for t in range(4)], 96, local_rank, warm=16, **cbr)
            s4 = resident_leg([synth.gradient(W, H, t) for t in range(N_DISTINCT)], 128, local_rank, warm=32, **cbr)
            content_legs = {"s2_noise_fps": s2["value"], "s2_bytes_per_picture": s2["bytes_per_picture"],
                            "s4_gradient_pan_fps": s4["value"], "s4_bytes_per_picture": s4["bytes_per_picture"],
                            "note": "same session settings as the headline leg (4K, CBR 20 Mbit/s), inputs resident; S2 = fresh uniform noise every picture "
                                    "(worst case: every macroblock runs the exhaustive search + refinement), S4 = smooth gradient panning 2 px/picture"}
        except Exception as e:
            content_legs = {"error": repr(e)}
        try:
            py_surface = python_surface_leg(frames, local_rank)
        except Exception as e:
            py_surface = {"error": repr(e)}
        try:      # how much of the GPU one free-running session leaves: two sessions on the same GPU, aggregate pictures/s
            import threading as _th
            res2 = [None, None]

            def _one(i):
                res2[i] = resident_leg(frames, 512, local_rank, warm=48, **cbr)
            ts = [_th.Thread(target=_one, args=(i,)) for i in range(2)]
            t0 = time.perf_counter()
            for t in ts:
                t.start()
            for t in ts:
                t.join()
            content_legs = dict(content_legs or {})
            content_legs["two_sessions_one_gpu_fps"] = sum(r["value"] for r in res2)
            content_legs["two_sessions_note"] = ("two independent sessions of the headline workload on ONE GPU, each device-timed over 512 pictures, "
                                                 "sum of the two rates (the headline `value` is one session per GPU, BASELINE configs[3])")
        except Exception as e:
            content_legs = dict(content_legs or {}, two_sessions_error=repr(e))
        try:      # the headline content with a 64-picture scroll cycle instead of 16 (2.1 GB resident): the restart picture, in which
            # nothing is predictable, is then 1 picture in 64
            long_frames = synth_frames(64)
            lc = resident_leg(long_frames, 512, local_rank, warm=64, **cbr)
            content_legs = dict(content_legs or {})
            content_legs["scroll_cycle64_fps"] = lc["value"]
            content_legs["scroll_cycle64_bytes_per_picture"] = lc["bytes_per_picture"]
            del long_frames
        except Exception as e:
            content_legs = dict(content_legs or {}, scroll_cycle64_error=repr(e))

    # ---------------- CPU baseline (rank 0, N=1 only; bounded sample) ------------------------------------------
    cpu = parity = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        try:
            one_fps, one_dt, _ = cpu_sample(frames, 2, threads=1)
            ref_aus = []
            all_fps, all_dt, cores = cpu_sample(frames, 24, threads=None, keep=ref_aus)
            parity = parity_leg(frames, ref_aus, local_rank)
            cpu = {"value": all_fps, "unit": "frames/s", "cores": cores, "kind": "port",
                   "sample": "1 IDR + 24 P pictures 3840x2160 (oracle CSC + encode, OpenMP over macroblock rows), IDR untimed; "
                             f"1 thread: {one_fps:.3f} frames/s over 2 P pictures",
                   "single_thread_value": one_fps,
                   "cgroup_cpu_quota": cpu_quota(), "note": "CPU restatement of this repo's encoder, not x264/videoconvert (absent from the image)",
                   "x264_anchor": x264_anchor(cores)}
        except Exception as e:  # the checker failing must not hide the GPU number
            cpu = {"value": None, "error": repr(e)}

    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, dump_aus)

    if rank == 0:
        line = {
            "metric": "4K frames/sec encoded", "value": value, "unit": "frames/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": t_ms / args.steps, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "u8", "data": "synthetic", "config": workload_config(FRAMES_PER_STEP),
            "e2e": {"value": e2e_value, "unit": "frames/s", "h2d_bytes_per_step": h2d_step, "d2h_bytes_per_step": d2h_step,
                    "wall_ms": e2e_wall_ms, "device_ms": e2e_dev_ms, "access_unit_bytes_per_frame": out_bytes[0] / max(1, n_frames),
                    "producer": "excluded: the pinned ring is pre-filled once (screen capture is out of scope, SURVEY.md §8b); the H2D copy of every "
                                "33 MB picture and the D2H copy of every access unit are inside the timed region; `python_surface` has a leg with a producer"},
            "gpu_launches": int(st["kernel_launches"]), "roofline": roofline, "cpu_baseline": cpu, "clocks": clk,
            "kernels_us": kern, "per_rank_ms_resident": per_rank_ms, "per_rank_wall_ms_resident": per_rank_wall_ms, "per_rank_ms_e2e": per_rank_e2e_ms,
            "per_rank_host_us_per_frame": {"resident": host_resident, "e2e": host_e2e,
                                           "keys": "output thread: wait_event (GPU not done yet), wait_job (idle), callback; submitter: wait_out_slot (back-pressure), wait_ring, submit (CUDA enqueue calls)"},
            "parity": parity, "idr": idr_legs, "content_legs": content_legs, "python_surface": py_surface, "per_rank_span_us": per_rank_span, "per_rank_inter_us": per_rank_inter, "per_rank_numa": per_rank_numa, "numa_node": numa, "wall_ms_resident": wall_ms, "target_fps": 240, "rtp_payloader": rtp_leg(sample_aus), "striped_mode": striped,
        }
        emit(line)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
