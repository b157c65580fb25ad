"""Time the batched loop-closure decision of many localisation clients.

    python tools/bench_decide.py [--clients 128 --steps 20 --warmup 5 --places 1000,10000,50000] [--no-fused] [--gps 10000]

1. lcd_decide_batch_dev (adjustLikelihood + the posterior of every client + the hypothesis selection) at `clients` clients over a map of
   `places` places (a chain graph with the default Bayes/PredictionLC), against `clients` sequential lcd_bayes_compute_posterior calls
   on the same map (each uploads and validates the neighbour tables on the host and returns the posterior to the host).
2. At the C2 shape (49 152 binary words, 10 000 signatures of 1000 words with their signature store, `clients` frames of 1000
   descriptors revisiting them): lcd_process_decide_batch_dev against lcd_process_batch_dev (quantise + score + verification of the
   raw-likelihood arg-max).  Rtabmap/LoopThr is 0 here, so that every frame's hypothesis is accepted and verified, as
   lcd_process_batch_dev verifies every frame; with the default 0.11 the decision may verify fewer frames and cost less.
3. With --gps N: at `clients` clients over N places with a GPS fix each (4 m apart on a straight line), lcd_decide_batch_dev against
   lcd_decide_gps_batch_dev with frames that carry no fix and with every frame carrying a fix, at radii (Rtabmap/LoopGPS with
   RGBD/LocalRadius) that keep about 1 %, 30 % and 100 % of the places; the calls alternate, twice each.
Device time with CUDA events after warm-up, over `steps` back-to-back calls; the sequential single-client calls are timed with the host
clock (they synchronise).  One JSON line on stdout, with the card's name and power limit read in this run."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from oracle.bayes_py import DEFAULT_PREDICTION_LC  # noqa: E402
from rtabmap_b200 import Engine, synth  # noqa: E402

W, S, F = 49152, 10000, 1000


def card():
    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=20)
        pl, clk = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        out.update(power_limit_w=float(pl), max_sm_clock_mhz=float(clk))
    except Exception as ex:  # the number still stands; say the limit was not read
        out["power_limit_w"] = f"not read: {ex}"
    return out


def time_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def chain_tables(n, levels):
    """CSR neighbour tables of a chain of n real places behind the virtual place (ids -1, 1..n), margins up to `levels`."""
    col_ptr = [0, 0]
    rows, lv = [], []
    for c in range(1, n + 1):
        for r in range(max(1, c - levels), min(n, c + levels) + 1):
            rows.append(r)
            lv.append(abs(r - c))
        col_ptr.append(len(rows))
    return np.array(col_ptr, np.int64), np.array(rows, np.int32), np.array(lv, np.int32)


def bench_posterior(B, n, steps, warmup, st):
    eng = Engine()
    lc = [float(np.float32(v)) for v in DEFAULT_PREDICTION_LC]
    levels = len(lc) - 2
    ids = np.concatenate([[-1], np.arange(1, n + 1)]).astype(np.int32)
    cp, rows, lv = chain_tables(n, levels)
    eng.clients_create(B)
    eng.clients_set_map(ids, cp, rows, lv, lc, 0.9)
    rng = np.random.default_rng(n)
    raw = (0.05 * rng.random((B, n))).astype(np.float32)
    raw[np.arange(B), rng.integers(0, n, B)] = 2.0
    d_like = torch.from_numpy(raw.reshape(-1)).cuda()
    d_post = torch.zeros(B * (n + 1), dtype=torch.float32, device="cuda")
    clients = np.arange(B, dtype=np.int32)
    flags = np.zeros(B, np.int32)
    dp = Engine.decide_params()
    torch.cuda.synchronize()
    ext = torch.cuda.ExternalStream(st(eng))
    with torch.cuda.stream(ext):
        ms = time_ms(lambda: eng.decide_batch_dev(d_like.data_ptr(), B, n, clients, flags, dp, d_post.data_ptr(), stream=st(eng)), steps, warmup)
    adj = eng.adjust_likelihood(raw)
    seq_steps = max(1, min(steps, 3))
    for b in range(min(B, 2)):  # warm-up
        eng.bayes_compute_posterior(ids, adj[b], cp, rows, lv, lc, 0.9)
    t0 = time.perf_counter()
    for _ in range(seq_steps):
        for b in range(B):
            eng.bayes_compute_posterior(ids, adj[b], cp, rows, lv, lc, 0.9)
    seq_ms = (time.perf_counter() - t0) * 1e3 / seq_steps
    state_mb = 2 * 4 * B * (n + 1) / 1e6  # re-keyed last posterior and unnormalised posterior, [place][client] floats
    return {"places": n, "decide_batch_ms": ms, "sequential_bayes_ms": seq_ms, "state_mb": state_mb, "speedup": seq_ms / ms}


def bench_gps(B, n, steps, warmup):
    eng = Engine()
    lc = [float(np.float32(v)) for v in DEFAULT_PREDICTION_LC]
    ids = np.concatenate([[-1], np.arange(1, n + 1)]).astype(np.int32)
    cp, rows, lv = chain_tables(n, len(lc) - 2)
    eng.clients_create(B)
    eng.clients_set_map(ids, cp, rows, lv, lc, 0.9)
    lat0, lon0, spacing = 46.78, -71.27, 4.0
    deg_e = 1.0 / (111320.0 * np.cos(np.radians(lat0)))
    gps = np.zeros((n, 5))
    gps[:, 0] = 1.0
    gps[:, 1] = lon0 + spacing * np.arange(n) * deg_e
    gps[:, 2] = lat0
    eng.clients_set_map_gps(ids[1:], gps)
    rng = np.random.default_rng(n)
    raw = (0.05 * rng.random((B, n))).astype(np.float32)
    raw[np.arange(B), rng.integers(0, n, B)] = 2.0
    fix = np.zeros((B, 5))
    fix[:, 0] = 2.0
    fix[:, 1] = lon0 + spacing * (n / 2 + rng.uniform(-0.1, 0.1, B) * n) * deg_e   # frames near the middle of the line
    fix[:, 2] = lat0
    fix[:, 4] = 2.0
    d_like = torch.from_numpy(raw.reshape(-1)).cuda()
    d_post = torch.zeros(B * (n + 1), dtype=torch.float32, device="cuda")
    d_cmp = torch.zeros(B * n, dtype=torch.uint8, device="cuda")
    clients = np.arange(B, dtype=np.int32)
    flags = np.zeros(B, np.int32)
    dp = Engine.decide_params()
    st = eng.stream
    length = spacing * n
    calls = {"decide_batch_ms": lambda: eng.decide_batch_dev(d_like.data_ptr(), B, n, clients, flags, dp, d_post.data_ptr(), stream=st),
             "gps_no_fix_ms": lambda: eng.decide_gps_batch_dev(d_like.data_ptr(), B, n, clients, flags, None, 10.0, dp, d_post.data_ptr(),
                                                               d_cmp.data_ptr(), stream=st)}
    for share in (0.01, 0.3, 1.0):
        r = share * length / 2 if share < 1 else 2 * length
        calls[f"gps_{int(share * 100)}pct_ms"] = (lambda r=r: eng.decide_gps_batch_dev(d_like.data_ptr(), B, n, clients, flags, fix, r, dp,
                                                                                          d_post.data_ptr(), d_cmp.data_ptr(), stream=st))
    res = {"places": n}
    ext = torch.cuda.ExternalStream(st)
    with torch.cuda.stream(ext):
        for _ in range(2):
            for k, fn in calls.items():
                res.setdefault(k, []).append(time_ms(fn, steps, warmup))
                if k.startswith("gps_") and k != "gps_no_fix_ms":
                    torch.cuda.synchronize()
                    res.setdefault(k.replace("_ms", "_kept"), float(d_cmp.float().mean()))
    return res


def bench_fused(B, steps, warmup):
    vocab = synth.make_binary_vocabulary(W, 32, 1)
    ids = np.arange(1, W + 1, dtype=np.int32)
    m = synth.make_map(ids, S, F, seed=2)
    store = synth.make_signature_store(vocab, ids, m)
    q, uv, places, _ = synth.make_query_frames_geo(store, m, B)
    eng = Engine(max_words=W, max_signatures=S + 2, max_queries=F, max_batch=B)
    eng.add_words(ids, vocab)
    eng.last_word_id = W
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    eng.set_ni(m.sig_ids, m.ni)
    eng.sig_add_batch(m.sig_ids, store.desc, store.xyz)
    lc = [float(np.float32(v)) for v in DEFAULT_PREDICTION_LC]
    map_ids = np.concatenate([[-1], m.sig_ids]).astype(np.int32)
    cp, rows, lv = chain_tables(S, len(lc) - 2)
    eng.clients_create(B)
    eng.clients_set_map(map_ids, cp, rows, lv, lc, 0.9)
    vp = Engine.verify_params(synth.CAMERA_K4)
    dp = Engine.decide_params(loop_thr=0.0)
    st = eng.stream
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_uv = torch.from_numpy(uv.reshape(-1)).cuda()
    d_s = torch.from_numpy(m.sig_ids).cuda()
    d_w = torch.zeros(B * F, dtype=torch.int32, device="cuda")
    d_l = torch.zeros(B * S, dtype=torch.float32, device="cuda")
    d_p = torch.zeros(B * (S + 1), dtype=torch.float32, device="cuda")
    clients = np.arange(B, dtype=np.int32)
    flags = np.zeros(B, np.int32)
    torch.cuda.synchronize()

    def plain():
        eng.process_batch_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, d_s.data_ptr(), S, S + 1, vp, d_w.data_ptr(), d_l.data_ptr(), stream=st)

    def decide():
        eng.process_decide_batch_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, S, S + 1, vp, clients, flags, dp, d_w.data_ptr(), d_l.data_ptr(),
                                     d_p.data_ptr(), stream=st)

    ext = torch.cuda.ExternalStream(st)
    res = {}
    with torch.cuda.stream(ext):
        for k in range(2):  # alternate the two calls
            res.setdefault("process_batch_ms", []).append(time_ms(plain, steps, warmup))
            res.setdefault("process_decide_batch_ms", []).append(time_ms(decide, steps, warmup))
    dec = eng.decide_fetch(B)
    res["accepted_frames"] = int((dec["status"] == 8).sum())
    res["accepted_is_place"] = int(((dec["status"] == 8) & (dec["loop_id"] == places)).sum())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clients", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--places", default="1000,10000,50000")
    ap.add_argument("--no-fused", action="store_true")
    ap.add_argument("--gps", type=int, default=0, help="places of the GPS-filter comparison (0: not run)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decide needs a CUDA device")
    res = {"clients": args.clients, "steps": args.steps, "warmup": args.warmup}
    res["posterior"] = [bench_posterior(args.clients, int(n), args.steps, args.warmup, lambda e: e.stream) for n in args.places.split(",")]
    if args.gps:
        res["gps"] = bench_gps(args.clients, args.gps, args.steps, args.warmup)
    if not args.no_fused:
        res["c2"] = bench_fused(args.clients, args.steps, args.warmup)
    res.update(card())
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
