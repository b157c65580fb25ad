"""Time lcd_epipolar_check_batch (EpipolarGeometry::check on the GPU) against cv2.findFundamentalMat on the host.

Workload: 128 pairs of 1000-keypoint signatures sharing 300-600 unique words, at inlier ratios 0.8, 0.5 and 0.3 (the last runs the
registrator's full 1000 iterations).  The kernel is timed with CUDA events recorded around each launch (lcd_profile_enable,
LCD_PROF_EPIPOLAR); the whole synchronous call (copies in, kernel, copies out) with the host clock.  The CPU leg runs
cv2.findFundamentalMat on every pair, one thread.  Prints one JSON line per inlier ratio, with the card's name and power limit read in
the same run."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from epipolar_cases import point_sets, signature_pair  # noqa: E402
from rtabmap_b200 import Engine  # noqa: E402

LCD_PROF_EPIPOLAR = 6


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def workload(n_pairs: int, inlier_ratio: float, seed: int):
    rng = np.random.default_rng(seed)
    cap = 1000
    out = [np.zeros((n_pairs, cap), np.int32), np.zeros((n_pairs, cap, 2), np.float32), np.full(n_pairs, cap, np.int32),
           np.zeros((n_pairs, cap), np.int32), np.zeros((n_pairs, cap, 2), np.float32), np.full(n_pairs, cap, np.int32)]
    pts = []
    for i in range(n_pairs):
        n = int(rng.integers(300, 601))
        p1, p2 = point_sets(n, 1 - inlier_ratio, "general", seed * 1000 + i)
        ia, ua, ib, ub = signature_pair(p1, p2, seed * 1000 + i + 500, extra=cap - n)
        out[0][i], out[1][i], out[3][i], out[4][i] = ia[:cap], ua[:cap], ib[:cap], ub[:cap]
        pts.append((p1, p2))
    return out, pts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import cv2

    eng = Engine(device=0)
    name = card()
    for ratio in (0.8, 0.5, 0.3):
        batch, pts = workload(args.pairs, ratio, int(ratio * 10))
        res = eng.epipolar_check_batch(*batch)  # warm-up: module load, shared-memory opt-in, scratch growth
        ts, ks = [], []
        for _ in range(args.reps):
            eng.profile_reset()
            eng.profile_enable(True)
            t0 = time.perf_counter()
            eng.epipolar_check_batch(*batch)
            ts.append((time.perf_counter() - t0) * 1e3)
            ms, launches = eng.profile_read(LCD_PROF_EPIPOLAR)
            eng.profile_enable(False)
            assert launches == 1
            ks.append(ms)
        t0 = time.perf_counter()
        for p1, p2 in pts:
            cv2.findFundamentalMat(p1, p2, cv2.FM_RANSAC, 3.0, 0.99)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        print(json.dumps({"workload": "epipolar_check_batch", "pairs": args.pairs, "inlier_ratio": ratio,
                          "kernel_ms_median": float(np.median(ks)), "call_ms_median": float(np.median(ts)), "cv2_ms_for_all_pairs": cpu_ms,
                          "mean_iterations": float(np.mean([r["iterations_run"] for r in res])),
                          "ok": int(sum(r["ok"] for r in res)), "card": name}))


if __name__ == "__main__":
    main()
