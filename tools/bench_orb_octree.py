"""Time detection + description per frame: ORB-OCTREE (Kp/DetectorStrategy=10) at ORB/ScaleFactor 2.0 x 3 levels and ORB-SLAM's
1.2 x 8 levels, beside FAST-ORB (2) and GFTT/ORB (8), in the same run.

Workload: batches of synthetic textured frames (rtabmap_b200.synth.make_image) at 640x480 and 1280x720, gray, no depth, Kp/MaxFeatures
1000, ORB/EdgeThreshold 19, FAST/Threshold 20, FAST/MinThreshold 7 (the reference defaults; ORB/NLevels 3 for FAST-ORB).  The
frames are already on the device; lcd_orb_detect_describe_dev runs on one stream and CUDA events recorded around `--reps` calls give
the time per call, divided by the batch size.  Prints one JSON line per (size, batch, detector), with the card's name and power limit
read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from rtabmap_b200 import Engine, synth  # noqa: E402
from rtabmap_b200.capi import DETECTOR_GFTT_ORB, DETECTOR_ORB, DETECTOR_ORB_OCTREE  # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32, 128])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_orb_octree needs a CUDA device")
    name = card()
    eng = Engine(device=0)
    lib, h = eng._lib, eng._h
    stream = torch.cuda.ExternalStream(eng.stream)  # the engine's own stream: the events must sit on the stream the kernels run on
    cap = 1000
    for height, width in ((480, 640), (720, 1280)):
        k4 = (500.0, 500.0, width / 2, height / 2)
        frames = np.stack([synth.make_image(height, width, 100 + i) for i in range(max(args.batches))])
        d_img = torch.from_numpy(frames).cuda()
        for batch in args.batches:
            d_kp = torch.empty((batch, cap, 6), dtype=torch.float32, device="cuda")
            d_desc = torch.empty((batch, cap, 32), dtype=torch.uint8, device="cuda")
            d_n = torch.empty(batch, dtype=torch.int32, device="cuda")
            for label, det, op in (("FAST-ORB", DETECTOR_ORB, Engine.orb_params(k4, n_features=cap)),
                                   ("GFTT/ORB", DETECTOR_GFTT_ORB, Engine.orb_params(k4, n_features=cap)),
                                   ("ORB-OCTREE 2.0x3", DETECTOR_ORB_OCTREE, Engine.orb_params(k4, n_features=cap)),
                                   ("ORB-OCTREE 1.2x8", DETECTOR_ORB_OCTREE, Engine.orb_params(k4, n_features=cap, n_levels=8, scale_factor=1.2))):
                if det == DETECTOR_ORB_OCTREE:
                    eng.set_detector_orb_octree(7)
                else:
                    eng.set_detector(det)

                def call():
                    rc = lib.lcd_orb_detect_describe_dev(h, batch, C.c_void_p(d_img.data_ptr()), width, height, 1, None, 0, C.byref(op), cap,
                                                         C.c_void_p(d_kp.data_ptr()), C.c_void_p(d_desc.data_ptr()), None, None,
                                                         C.c_void_p(d_n.data_ptr()), C.c_void_p(stream.cuda_stream))
                    if rc != 0:
                        raise RuntimeError(lib.lcd_last_error(h).decode())

                torch.cuda.synchronize()  # the uploads above ran on torch's stream
                for _ in range(args.warmup):
                    call()
                torch.cuda.synchronize()
                if eng.orb_overflow():
                    raise RuntimeError("candidate list truncated")
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record(stream)
                for _ in range(args.reps):
                    call()
                t1.record(stream)
                t1.synchronize()
                ms = t0.elapsed_time(t1) / args.reps
                print(json.dumps({"size": f"{width}x{height}", "batch": batch, "detector": label,
                                  "ms_per_call": round(ms, 4), "ms_per_frame": round(ms / batch, 4),
                                  "mean_keypoints": round(float(d_n.float().mean().item()), 1), "gpu": name}), flush=True)


if __name__ == "__main__":
    main()
