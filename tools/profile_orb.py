"""Where the time of the FAST-ORB detect stage goes, per kernel and per stream, at the benchmark's frame size and several batch sizes.

Workload: bench.py's world and query frames (rtabmap_b200.synth, 640x480 BGR + 16-bit depth, the place images detected by the engine's
own ORB), Kp/MaxFeatures 1000, 3 levels, depth mask and 3-D lifting, through lcd_orb_detect_describe_dev on the engine's stream.

Per batch size it prints one JSON line with
  * `ms_per_call`: CUDA events around `--reps` calls with the profiler off;
  * `kernels`: a separate torch.profiler run of `--prof-reps` calls, every kernel's device time summed per (name, stream) and divided by
    the number of calls; `streams`: the busy time per stream (level 0 runs on the caller's stream, levels 1-2 and the blur on side
    streams), so the critical path of the stage is the caller's stream plus its waits;
  * `cand_gpu`: the engine's FAST candidate counts per level (mean and max over the frames), read back from its candidate counters;
  * `cand_cv2_estimate`: an ESTIMATE of the same counts on the host, cv2.FastFeatureDetector (threshold 20, non-max suppression) on each
    level of the oracle's pyramid (INTER_LINEAR_EXACT halving), with the depth mask and the ORB/EdgeThreshold border applied.
The first line names the card, its power limit and its maximum SM clock, read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import tempfile
from collections import defaultdict
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from rtabmap_b200 import Engine, synth  # noqa: E402

W, H, FEATS, N_PLACES, WORDS, SIGS = 640, 480, 1000, 50, 49152, 10000  # bench.py's headline configuration
KCAM = synth.CAMERA_K4


def card() -> dict:
    q = "name,power.limit,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in line.split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError):
        return {"name": "unknown"}


def cv2_candidates(img, dep, n_levels=3, thr=20, edge=19):
    """FAST corners per level of one frame as cv::ORB would find them before retainBest: an estimate (the pyramid and filters are restated
    here, not taken from OpenCV's ORB)"""
    import cv2

    from oracle import feature2d_py as f2d

    gray = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    mask = f2d.depth_mask(dep, f2d.OrbParams())
    fast = cv2.FastFeatureDetector_create(thr, True)
    out = []
    for lv in range(n_levels):
        if lv:
            size = (gray.shape[1] // 2, gray.shape[0] // 2)
            gray = cv2.resize(gray, size, interpolation=cv2.INTER_LINEAR_EXACT)
            mask = cv2.threshold(cv2.resize(mask, size, interpolation=cv2.INTER_LINEAR_EXACT), 254, 0, cv2.THRESH_TOZERO)[1]
        h, w = gray.shape
        n = 0
        for k in fast.detect(gray):
            x, y = int(round(k.pt[0])), int(round(k.pt[1]))
            n += edge <= x < w - edge and edge <= y < h - edge and mask[y, x] != 0
        out.append(n)
    return out


def bench_frames(eng, n_frames):
    op = Engine.orb_params(KCAM, n_features=FEATS)
    world = synth.make_place_world(lambda img, dep: eng.orb_detect_describe(img[None], dep[None], op, cap=FEATS)[0], N_PLACES, WORDS, SIGS, FEATS, H, W)
    imgs, deps, _ = synth.make_view_frames(world, 3 * n_frames, seed=3, mode="revisit")  # bench.py's pool of the first rank; its first batch
    return imgs[:n_frames], deps[:n_frames]


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 32, 64, 128])
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--prof-reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cv2-frames", type=int, default=32, help="frames of the batch whose candidate counts cv2 estimates")
    ap.add_argument("--out", default=None, help="directory for the profiler traces (default: a temporary directory)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_orb needs a CUDA device")
    out_dir = Path(args.out or tempfile.mkdtemp(prefix="profile_orb_"))
    out_dir.mkdir(parents=True, exist_ok=True)
    print(json.dumps({"card": card()}), flush=True)
    eng = Engine(device=0, max_queries=FEATS, max_batch=max(args.batches))
    lib, h = eng._lib, eng._h
    op = Engine.orb_params(KCAM, n_features=FEATS)
    imgs, deps = bench_frames(eng, max(args.batches))
    est = np.array([cv2_candidates(imgs[i], deps[i]) for i in range(min(args.cv2_frames, len(imgs)))])
    stream = torch.cuda.ExternalStream(eng.stream)
    d_img = torch.from_numpy(imgs).cuda()
    d_dep = torch.from_numpy(deps.view(np.int16)).cuda()
    for batch in args.batches:
        d_kp = torch.empty((batch, FEATS, 6), dtype=torch.float32, device="cuda")
        d_desc = torch.empty((batch, FEATS, 32), dtype=torch.uint8, device="cuda")
        d_xyz = torch.empty((batch, FEATS, 3), dtype=torch.float32, device="cuda")
        d_uv = torch.empty((batch, FEATS, 2), dtype=torch.float32, device="cuda")
        d_n = torch.empty(batch, dtype=torch.int32, device="cuda")

        def call():
            rc = lib.lcd_orb_detect_describe_dev(h, batch, C.c_void_p(d_img.data_ptr()), W, H, 3, C.c_void_p(d_dep.data_ptr()), 1, C.byref(op), FEATS,
                                                 C.c_void_p(d_kp.data_ptr()), C.c_void_p(d_desc.data_ptr()), C.c_void_p(d_xyz.data_ptr()),
                                                 C.c_void_p(d_uv.data_ptr()), C.c_void_p(d_n.data_ptr()), C.c_void_p(stream.cuda_stream))
            if rc != 0:
                raise RuntimeError(lib.lcd_last_error(h).decode())

        torch.cuda.synchronize()
        for _ in range(args.warmup):
            call()
        torch.cuda.synchronize()
        if eng.orb_overflow():
            raise RuntimeError("candidate list truncated")
        counts = eng.debug_orb_buffer(4, batch * 3 * 4, np.int32).reshape(batch, 3)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        for _ in range(args.reps):
            call()
        t1.record(stream)
        t1.synchronize()
        ms = t0.elapsed_time(t1) / args.reps

        trace = out_dir / f"orb_b{batch}.pt.trace.json"
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.prof_reps):
                call()
            torch.cuda.synchronize()
        prof.export_chrome_trace(str(trace))
        ev = [e for e in json.loads(trace.read_text())["traceEvents"] if e.get("cat") == "kernel"]
        per = defaultdict(float)
        busy = defaultdict(float)
        for e in ev:
            name = e["name"].split("(")[0].split("<")[0]
            sid = e.get("args", {}).get("stream", -1)
            per[(name, sid)] += e["dur"] / 1e3 / args.prof_reps
            busy[sid] += e["dur"] / 1e3 / args.prof_reps
        span = (max(e["ts"] + e["dur"] for e in ev) - min(e["ts"] for e in ev)) / 1e3 / args.prof_reps if ev else 0.0
        print(json.dumps({
            "batch": batch, "ms_per_call": round(ms, 4), "ms_per_frame": round(ms / batch, 5),
            "profiled_span_ms_per_call": round(span, 4),
            "streams": {str(s): round(v, 4) for s, v in sorted(busy.items(), key=lambda kv: -kv[1])},
            "kernels": [{"kernel": n, "stream": s, "ms_per_call": round(v, 4)} for (n, s), v in sorted(per.items(), key=lambda kv: -kv[1])],
            "cand_gpu": {"mean": counts.mean(0).round(1).tolist(), "max": counts.max(0).tolist()},
            "cand_cv2_estimate": {"frames": len(est), "mean": est.mean(0).round(1).tolist(), "max": est.max(0).tolist()},
            "mean_keypoints": round(float(d_n.float().mean().item()), 1)}), flush=True)


if __name__ == "__main__":
    main()
