"""Time lcd_process_frames_dev with Memory::createSignature's split (lcd_quantize_limit_set, Kp/MaxFeatures 500 of 1000 detected) against
the same call without it, alternating the two in one process.

Workload: bench.py's C2 world (49 152 words, 10 000 signatures, 1000 ORB features per 640x480 RGB-D frame), batches of 128 revisit
frames already on the device, verification on.  Each round times `--reps` calls of each setting with CUDA events on the engine's stream;
the rounds alternate the settings.  A second pass reads the engine's per-stage timers (lcd_profile_*) for both settings: the dictionary
search and the resolve stage see k rows per frame instead of the detection count, verification sees every row in both.  With
--profile-select, a separate run times the selection and expansion kernels alone under torch.profiler.  Prints JSON lines, with the
card's name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from rtabmap_b200 import Engine, synth  # noqa: E402

W_WORDS, S_SIGS, F_FEATS, N_PLACES, IMG_W, IMG_H = 49152, 10000, 1000, 50, 640, 480
KCAM = (500.0, 500.0, IMG_W / 2 - 0.5, IMG_H / 2 - 0.5)
STAGES = {"nn": 0, "resolve": 1, "score": 2, "match": 3, "pnp": 4, "orb": 5}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--limit", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--profile-select", action="store_true", help="time the selection kernel alone under torch.profiler (separate run)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_quantize_limit needs a CUDA device")
    name = card()
    B = args.batch
    eng = Engine(device=0, max_words=W_WORDS + 1024, max_signatures=S_SIGS + 16, max_queries=F_FEATS, max_batch=B)
    op = Engine.orb_params(KCAM, n_features=F_FEATS)
    vp = Engine.verify_params(KCAM, image_size=(IMG_W, IMG_H))
    world = synth.make_place_world(lambda im, dp: eng.orb_detect_describe(im[None], dp[None], op, cap=F_FEATS)[0], N_PLACES, W_WORDS, S_SIGS,
                                   F_FEATS, IMG_H, IMG_W)
    sm = world.smap
    eng.add_words(world.word_ids, world.vocab)
    eng.last_word_id = int(world.word_ids.max())
    eng.update()
    eng.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    eng.set_ni(sm.sig_ids, sm.ni)
    eng.sig_add_batch(sm.sig_ids, world.store.desc, world.store.xyz, sm.ni)
    imgs, deps, _ = synth.make_view_frames(world, B, seed=3)
    d_img = torch.from_numpy(imgs).cuda()
    d_dep = torch.from_numpy(deps.view(np.int16)).cuda()
    d_sig = torch.from_numpy(sm.sig_ids).cuda()
    d_w = torch.zeros(B * F_FEATS, dtype=torch.int32, device="cuda")
    d_l = torch.zeros(B * S_SIGS, dtype=torch.float32, device="cuda")
    stream = torch.cuda.ExternalStream(eng.stream)
    settings = {"off": (0, 0.0, 0), f"limit{args.limit}": (args.limit, 0.5, args.limit)}

    def step():
        eng.process_frames_dev(d_img.data_ptr(), B, IMG_W, IMG_H, 3, d_dep.data_ptr(), 1, op, d_sig.data_ptr(), S_SIGS, S_SIGS + 1, vp,
                               d_w.data_ptr(), d_l.data_ptr())

    if args.profile_select:
        from torch.profiler import ProfilerActivity, profile

        eng.set_quantize_limit(*settings[f"limit{args.limit}"])
        k = args.limit
        d_kp = torch.zeros((B, F_FEATS, 24), dtype=torch.uint8, device="cuda")
        d_desc = torch.zeros((B, F_FEATS, 32), dtype=torch.uint8, device="cuda")
        d_n = torch.zeros(B, dtype=torch.int32, device="cuda")
        d_q = torch.zeros((B, k, 32), dtype=torch.uint8, device="cuda")
        d_idx = torch.zeros((B, k), dtype=torch.int32, device="cuda")
        d_nq = torch.zeros(B, dtype=torch.int32, device="cuda")
        d_wq = torch.ones((B, k), dtype=torch.int32, device="cuda")
        import ctypes

        eng._check(eng._lib.lcd_orb_detect_describe_dev(eng.handle, B, d_img.data_ptr(), IMG_W, IMG_H, 3, d_dep.data_ptr(), 1, ctypes.byref(op),
                                                        F_FEATS, d_kp.data_ptr(), d_desc.data_ptr(), None, None, d_n.data_ptr(), None))
        eng.synchronize()
        with torch.cuda.stream(stream):
            for _ in range(5):
                eng.limit_keypoints_dev(B, F_FEATS, d_kp.data_ptr(), d_n.data_ptr(), d_desc.data_ptr(), d_q.data_ptr(), d_idx.data_ptr(), d_nq.data_ptr())
            eng.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps * 10):
                    eng.limit_keypoints_dev(B, F_FEATS, d_kp.data_ptr(), d_n.data_ptr(), d_desc.data_ptr(), d_q.data_ptr(), d_idx.data_ptr(),
                                            d_nq.data_ptr())
                    eng.word_ids_expand_dev(B, F_FEATS, k, d_n.data_ptr(), d_idx.data_ptr(), d_nq.data_ptr(), d_wq.data_ptr(), d_w.data_ptr())
                eng.synchronize()
        kern = {}
        for ev in prof.key_averages():
            for tag in ("limit_keypoints_kernel", "word_ids_expand_kernel"):
                if tag in ev.key:
                    t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                    kern[tag] = {"calls": ev.count, "us_per_call": t / max(ev.count, 1), "us_per_frame": t / max(ev.count, 1) / B}
        print(json.dumps({"bench": "quantize_limit_select", "card": name, "batch": B, "detected": F_FEATS, "k": k, "kernels": kern}), flush=True)
        return

    # warm-up of both settings (module load, buffer growth, the tensor-core image of the dictionary)
    for lim in settings.values():
        eng.set_quantize_limit(*lim)
        for _ in range(3):
            step()
    eng.synchronize()
    times = {s: [] for s in settings}
    with torch.cuda.stream(stream):
        for r in range(args.rounds):
            for s, lim in (settings.items() if r % 2 == 0 else reversed(list(settings.items()))):
                eng.set_quantize_limit(*lim)
                step()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                for _ in range(args.reps):
                    step()
                b.record(stream)
                b.synchronize()
                times[s].append(a.elapsed_time(b) / args.reps)
    # per-stage device time (the engine's own event timers), one pass per setting
    stages = {}
    for s, lim in settings.items():
        eng.set_quantize_limit(*lim)
        eng.profile_enable(True)
        eng.profile_reset()
        for _ in range(args.reps):
            step()
        stages[s] = {k: eng.profile_read(v)[0] / args.reps for k, v in STAGES.items()}
        eng.profile_enable(False)
    hyp, _ = eng.process_fetch(B)
    for s in settings:
        med = statistics.median(times[s])
        print(json.dumps({"bench": "quantize_limit", "card": name, "setting": s, "limit": settings[s], "batch": B, "words": W_WORDS,
                          "signatures": S_SIGS, "detected": F_FEATS, "ms_per_step_median": med, "ms_per_step_rounds": times[s],
                          "us_per_frame": med * 1000.0 / B, "stage_ms_per_step": stages[s]}), flush=True)
    print(json.dumps({"bench": "quantize_limit_speedup", "card": name,
                      "off_over_limit": statistics.median(times["off"]) / statistics.median(times[f"limit{args.limit}"]),
                      "frames_with_hypothesis": int((hyp > 0).sum())}), flush=True)


if __name__ == "__main__":
    main()
