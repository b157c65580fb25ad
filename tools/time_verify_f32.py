"""Time geometric verification on float-descriptor engines: 128 pairs of 1000 descriptors per side at 64-D and 128-D through
lcd_verify_batch (match and PnP times from the engine's profile classes, as tools/time_verify.py reports them), and the fused
lcd_verify_top_dev against a 10 000-signature float store (2.6 GB at 64-D) with the FROM-dictionary cache cold and warm.
Prints one JSON line per measurement, with the card's name and power limit."""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
from rtabmap_b200 import Engine  # noqa: E402
from rtabmap_b200.capi import LCD_DESC_F32  # noqa: E402
from test_gpu_verify_f32 import IMG, K4, WIN, make_scene  # noqa: E402

B, N, REPS = 128, 1000, 5


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": q.stdout.strip()}


def scenes(dim, seed):
    rng = np.random.default_rng(seed)
    F = np.zeros((B, N, dim), np.float32)
    T = np.zeros((B, N, dim), np.float32)
    X = np.zeros((B, N, 3), np.float32)
    U = np.zeros((B, N, 2), np.float32)
    for i in range(B):
        F[i], X[i], T[i], U[i], _ = make_scene(rng, N, N, dim)
    return F, X, T, U


def time_batch(dim, info):
    F, X, T, U = scenes(dim, dim)
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=dim)
    eng.profile_enable(True)
    for repeat in (False, True):
        for _ in range(2):
            out = eng.verify_batch(F, X, T, U, K4, image_size=IMG, repeat_once=repeat, guess_win_size=WIN)
        eng.profile_reset()
        t0 = time.perf_counter()
        for _ in range(REPS):
            out = eng.verify_batch(F, X, T, U, K4, image_size=IMG, repeat_once=repeat, guess_win_size=WIN)
        dt = (time.perf_counter() - t0) / REPS
        m, p = eng.profile_read(3), eng.profile_read(4)
        # the match class holds the first-pass matching and, with Reg/RepeatOnce, the guess pass; PnP runs once per pass
        print(json.dumps({"call": "verify_batch", "dim": dim, "pairs": B, "desc_per_side": N, "repeat_once": repeat, "wall_ms": round(dt * 1e3, 3),
                          "match_ms": round(m[0] / REPS, 4), "pnp_ms": round(p[0] / REPS, 4), "ok": sum(o["ok"] for o in out), **info}), flush=True)
    eng.close()


def time_fused(dim, n_sigs, info):
    import torch

    F, X, T, U = scenes(dim, 7 + dim)
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=dim)
    ids = np.arange(1, n_sigs + 1, dtype=np.int32)
    chunk = 500
    for s0 in range(0, n_sigs, chunk):
        k = np.arange(s0, min(n_sigs, s0 + chunk)) % B
        eng.sig_add_batch(ids[s0:s0 + len(k)], F[k], X[k])
    # frame b is registered against signature pick[b], whose row holds scene b's FROM side
    pick = np.array([1 + b + B * ((b * 37) % (n_sigs // B)) for b in range(B)], np.int32)
    like = np.zeros((B, n_sigs), np.float32)
    like[np.arange(B), pick - 1] = 1.0
    d_l = torch.from_numpy(like.reshape(-1)).cuda()
    d_s = torch.from_numpy(ids).cuda()
    d_q = torch.from_numpy(T.reshape(-1)).cuda()
    d_uv = torch.from_numpy(U.reshape(-1)).cuda()
    vp = Engine.verify_params(K4, image_size=IMG, repeat_once=True, guess_win_size=WIN)
    torch.cuda.synchronize()

    def run():
        t0 = time.perf_counter()
        eng.verify_top_dev(d_q.data_ptr(), d_uv.data_ptr(), B, N, d_l.data_ptr(), d_s.data_ptr(), n_sigs, vp)
        hyp, res = eng.process_fetch(B)
        return time.perf_counter() - t0, hyp, res

    run()
    cold, warm = [], []
    for _ in range(REPS):
        eng.sig_add_batch(pick, F[np.arange(B)], X[np.arange(B)])  # rewritten rows: their cached dictionaries are stale
        torch.cuda.synchronize()
        cold.append(run()[0])
        dt, hyp, res = run()
        warm.append(dt)
    assert np.array_equal(hyp, pick)
    print(json.dumps({"call": "verify_top_dev", "dim": dim, "store_signatures": n_sigs, "store_gb": round(n_sigs * N * dim * 4 / 1e9, 2),
                      "frames": B, "cold_ms": round(float(np.median(cold)) * 1e3, 3), "warm_ms": round(float(np.median(warm)) * 1e3, 3),
                      "ok": sum(r["ok"] for r in res), **info}), flush=True)
    eng.close()


if __name__ == "__main__":
    info = card()
    for dim in (64, 128):
        time_batch(dim, info)
    time_fused(64, 10000, info)
