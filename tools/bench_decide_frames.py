"""Frames/s of the service call with the decision (lcd_process_frames_decide_submit / _wait) against the call without it
(lcd_process_frames_submit / _wait) on the same frame pool, at bench.py's configuration (BASELINE configs[1]: 640x480 RGB-D, ORB 1000
keypoints, 49 152 words, 10 000 places) and batch size, two batches in flight.  Four arms, alternated round by round in one run:

    plain      lcd_process_frames_submit (arg-max of the raw likelihood, verified)
    decide     lcd_process_frames_decide_submit, no optional stage
    decide+    the same with the GPS filter, the epipolar check and proximity detection by space on
    mixed      the two calls alternated batch by batch (plain, decide, plain, ...)

Prints the card's name and power limit beside the numbers, and one JSON line.  Needs a GPU.
    python tools/bench_decide_frames.py [--batch 128] [--steps 30] [--rounds 3]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from rtabmap_b200 import Engine, dbio, graph, synth  # noqa: E402
from rtabmap_b200.capi import DECISION_DTYPE, EpipolarParams, EpipolarResult, ProximityResult, VerifyResult  # noqa: E402

W_WORDS, S_SIGS, F_FEATS, N_PLACES, IMG_W, IMG_H = 49152, 10000, 1000, 50, 640, 480   # bench.py's configs[1]
KCAM = (525.0, 525.0, 320.0, 240.0)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def pinned(ctype):
    """a ctypes array in pinned host memory: lcd_process_frames_submit copies the verification records straight into it, and a device ->
    host copy into pageable memory would hold the submit until the batch is done"""
    import torch

    buf = torch.zeros(ctypes.sizeof(ctype), dtype=torch.uint8).pin_memory()
    arr = ctype.from_address(buf.data_ptr())
    arr._buf = buf
    return arr


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pool", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing is measured")
    B = args.batch
    eng = Engine(desc_dim=32, max_words=W_WORDS + 65536, max_signatures=S_SIGS + 128, max_queries=F_FEATS, max_batch=B)
    op = Engine.orb_params(KCAM, n_features=F_FEATS)
    vp = Engine.verify_params(KCAM, image_size=(IMG_W, IMG_H))
    t0 = time.time()
    world = synth.make_place_world(lambda im, dp: eng.orb_detect_describe(im[None], dp[None], op, cap=F_FEATS)[0], N_PLACES, W_WORDS, S_SIGS,
                                   F_FEATS, IMG_H, IMG_W)
    imgs, deps, places = synth.make_view_frames(world, B * args.pool, seed=3, mode="revisit")
    sm = world.smap
    eng.add_words(world.word_ids, world.vocab)
    eng.last_word_id = W_WORDS
    eng.update()
    eng.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    eng.set_ni(sm.sig_ids, sm.ni)
    kps = [eng.orb_detect_describe(world.images[p][None], world.depths[p][None], op, cap=F_FEATS)[0][0] for p in range(N_PLACES)]
    for s0 in range(0, S_SIGS, 1000):
        sl = slice(s0, s0 + 1000)
        eng.sig_add_batch(sm.sig_ids[sl], world.store.desc[sl], world.store.xyz[sl], sm.ni[sl])
        uv = np.zeros((1000, F_FEATS, 2), np.float32)
        for i, p in enumerate(world.sig_place[sl]):
            uv[i, :len(kps[int(p)])] = kps[int(p)][:, :2]
        eng.sig_words_add_batch(sm.sig_ids[sl], sm.sig_words[sl], uv, sm.ni[sl])
    # the map: places chained by neighbour links in id order, 0.5 m apart, every place with a GPS fix
    ids = [int(s) for s in sm.sig_ids]
    a, b = np.array(ids[:-1], np.int32), np.array(ids[1:], np.int32)
    eye = np.tile(np.eye(4, dtype=np.float32)[:3], (2 * len(a), 1, 1))
    links = dbio.Links(np.concatenate([a, b]), np.concatenate([b, a]), np.full(2 * len(a), graph.NEIGHBOR, np.int32), eye)
    lc = graph.DEFAULT_PREDICTION_LC
    tab = graph.prediction_tables(ids, graph.bayes_neighbors(ids, links, len(lc) - 1))
    eng.clients_create(B)
    eng.clients_set_map(tab[0], tab[1], tab[2], tab[3], lc, 0.9)
    poses = np.tile(np.eye(4, dtype=np.float32)[:3], (len(ids), 1, 1))
    poses[:, 0, 3] = 0.5 * np.arange(len(ids))
    eng.clients_set_map_poses(ids, poses, *graph.neighbor_links(ids, links))
    eng.clients_set_map_gps(ids, np.array([(1.0, -73.6 + 5e-6 * i, 45.5, 30.0, 2.0) for i in range(len(ids))]))
    print(f"set-up {time.time() - t0:.1f}s", file=sys.stderr)

    ns = len(ids)
    sig = np.array(ids, np.int32)
    h_img = [torch.from_numpy(np.ascontiguousarray(imgs[k * B:(k + 1) * B])).pin_memory() for k in range(args.pool)]
    h_dep = [torch.from_numpy(np.ascontiguousarray(deps[k * B:(k + 1) * B]).view(np.int16)).pin_memory() for k in range(args.pool)]
    dp = Engine.decide_params()
    clients = np.arange(B, dtype=np.int32)
    flags = np.zeros(B, np.int32)
    fpose = poses[np.clip(places.reshape(args.pool, B) * (S_SIGS // N_PLACES), 0, ns - 1)]
    fgps = [np.array([(1.0, -73.6 + 5e-6 * int(p) * (S_SIGS // N_PLACES), 45.5, 30.0, 2.0) for p in places[k * B:(k + 1) * B]])
            for k in range(args.pool)]
    ep = EpipolarParams(8, 3.0, 0.99)
    pp = Engine.proximity_params(vp, local_radius=2.0)
    stages_all = [Engine.decide_stages(B, fgps[k], 10.0, ep, pp, fpose[k], np.ones(B, np.int32)) for k in range(args.pool)]
    out = [dict(nkp=torch.zeros(B, dtype=torch.int32).pin_memory().numpy(), words=torch.zeros(B * F_FEATS, dtype=torch.int32).pin_memory().numpy(),
                like=torch.zeros(B * ns, dtype=torch.float32).pin_memory().numpy(), hyp=torch.zeros(B, dtype=torch.int32).pin_memory().numpy(),
                dec=np.zeros(B, DECISION_DTYPE), res=pinned(VerifyResult * B), epi=(EpipolarResult * B)(), prox=(ProximityResult * B)())
           for _ in range(2)]

    def submit(kind, k):
        o = out[k & 1]
        im, de = h_img[k % args.pool].numpy(), h_dep[k % args.pool].numpy().view(np.uint16)
        if kind == "plain":
            eng.process_frames_submit(im, de, op, sig, ns + 1, vp, o["nkp"], o["words"], o["like"], o["hyp"], o["res"])
        else:
            st = stages_all[k % args.pool] if kind == "decide+" else None
            eng.process_frames_decide_submit(im, de, op, ns, ns + 1, vp, clients, flags, dp, st, o["nkp"], o["words"], o["like"], o["dec"],
                                             o["res"], o["epi"] if st else None, o["prox"] if st else None)

    def run(kind, steps):
        kinds = ["plain", "decide"] * steps if kind == "mixed" else [kind] * steps
        t = time.perf_counter()
        for k, kk in enumerate(kinds[:steps]):
            submit(kk, k)
            if k >= 1:
                eng.process_frames_wait()
        eng.process_frames_wait()
        return steps * B / (time.perf_counter() - t)

    arms = ("plain", "decide", "decide+", "mixed")
    for kind in arms:
        run(kind, args.warmup)
    rates = {kind: [] for kind in arms}
    for _ in range(args.rounds):
        for kind in arms:
            rates[kind].append(run(kind, args.steps))
    gpu = card()
    for kind in arms:
        r = rates[kind]
        print(f"{kind:8s} {min(r):9.0f} .. {max(r):9.0f} frames/s  ({gpu})")
    print(json.dumps({"gpu": gpu, "batch": B, "steps": args.steps, "rounds": args.rounds, "frames_per_s": rates}))


if __name__ == "__main__":
    main()
