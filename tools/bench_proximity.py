"""Time proximity detection by space (lcd_decide_proximity_dev) for 128 localisation clients at 10 000 and 50 000 places.

Reports, from a host clock around work that ends in a device synchronise, over --reps runs after --warmup runs, the median of:
  decide_verify_ms            lcd_decide_batch_dev + lcd_verify_decided_dev
  decide_proximity_verify_ms  the same with lcd_decide_proximity_dev between them
  proximity_call_ms           lcd_decide_proximity_dev alone
  candidate_kernel_ms         proximity_paths_kernel alone, from CUDA events around its launch (LCD_PROF_PROXIMITY), mean per call
  registrations_ms            the call's matching and PnP kernels (LCD_PROF_MATCH + LCD_PROF_PNP), mean per call
The scene is the one of tests/test_gpu_proximity.py.  Prints one JSON line per map size, with the GPU's name, power limit and clock."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--places", type=int, nargs="+", default=[10000, 50000])
    ap.add_argument("--clients", type=int, default=128)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", type=str, default="")
    args = ap.parse_args()
    import torch

    import test_gpu_proximity as T
    from rtabmap_b200 import Engine, synth

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    vocab = synth.make_binary_vocabulary(49152, 32, 1)
    wid = np.arange(1, 49153, dtype=np.int32)
    m = synth.make_map(wid, T.S, T.F, seed=2)
    st = synth.make_signature_store(vocab, wid, m)
    q, uv, places, _ = synth.make_query_frames_geo(st, m, 128)
    world = (vocab, wid, m, st, q, uv, places)
    *_, q, uv, places = world
    B, F = args.clients, T.F
    lines = []
    for n in args.places:
        ids, poses, nbr, ptr, flat = T.scene(n)
        eng = T.make_engine(world, n, B)
        T.set_map(eng, ids)
        eng.clients_set_map_poses(ids, poses, ptr, flat)
        fp, raw, flags, enabled = T.frames(world, ids, poses, B, seed=1)
        d_like = torch.from_numpy(raw.reshape(-1)).cuda()
        d_q = torch.from_numpy(q[: B * F].reshape(-1)).cuda()
        d_uv = torch.from_numpy(uv[: B * F].reshape(-1)).cuda()
        dp = Engine.decide_params()
        vp = Engine.verify_params(synth.CAMERA_K4)
        pp = Engine.proximity_params(vp)
        clients = np.arange(B)
        torch.cuda.synchronize()

        def step(prox, only_prox=False):
            eng.clients_create(B)
            eng.decide_batch_dev(d_like.data_ptr(), B, n, clients, flags, dp)
            eng.synchronize()
            t0 = time.perf_counter()
            if prox:
                eng.decide_proximity_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, fp, enabled, pp)
            if only_prox:
                eng.synchronize()
                return (time.perf_counter() - t0) * 1e3
            eng.verify_decided_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, vp)

        res = {}
        for name, prox in (("decide_verify", False), ("decide_proximity_verify", True)):
            for _ in range(args.warmup):
                step(prox)
            eng.synchronize()
            ts = []
            for _ in range(args.reps):
                eng.clients_create(B)   # every rep decides from the same empty client state
                eng.synchronize()
                t0 = time.perf_counter()
                eng.decide_batch_dev(d_like.data_ptr(), B, n, clients, flags, dp)
                if prox:
                    eng.decide_proximity_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, fp, enabled, pp)
                eng.verify_decided_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, vp)
                eng.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            res[name + "_ms"] = float(np.median(ts))
        # the candidate kernel and the registrations from the events the profile hooks record around their launches
        eng.profile_reset()
        eng.profile_enable(True)
        ts = []
        for _ in range(args.reps):
            ts.append(step(True, only_prox=True))
        match_ms, _ = eng.profile_read(3)
        pnp_ms, _ = eng.profile_read(4)
        cand_ms, launches = eng.profile_read(7)
        eng.profile_enable(False)
        assert launches == args.reps
        res["proximity_call_ms"] = float(np.median(ts))
        res["registrations_ms"] = float((match_ms + pnp_ms) / args.reps)
        res["candidate_kernel_ms"] = float(cand_ms / args.reps)
        rec = eng.proximity_fetch(B)
        line = dict(places=n, clients=B, gpu=gpu, mean_nearest=float(np.mean([r["n_nearest"] for r in rec])),
                    mean_paths=float(np.mean([r["n_paths"] for r in rec])), attempts=int(sum(r["n_attempts"] for r in rec)), **res)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
