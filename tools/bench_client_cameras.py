"""Frames/s of the service call with the decision (lcd_process_frames_decide_submit / _wait) when every localisation client brings its
own camera (lcd_clients_set_cameras), at bench.py's C2 world (BASELINE configs[1]: 640x480 RGB-D, ORB 1000 keypoints, 49 152 words,
10 000 places) and batch size, two batches in flight.  Three arms, alternated round by round in one run:

    shared     one camera for every frame: no client camera, the call's lcd_orb_params / lcd_verify_params K
    distinct   128 distinct cameras (fx 480-640, principal point within 20 px, the optical rotation and offsets up to 0.5 m), one call
    per_client what a service does without client cameras: one one-frame call per client with its own K, two calls in flight

Prints the card's name and power limit beside the numbers, and one JSON line.  Needs a GPU.
    python tools/bench_client_cameras.py [--batch 128] [--steps 20] [--rounds 3]"""
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
from rtabmap_b200.capi import DECISION_DTYPE, OPTICAL_ROTATION, VerifyResult, camera_model  # noqa: E402

W_WORDS, S_SIGS, F_FEATS, N_PLACES, IMG_W, IMG_H = 49152, 10000, 1000, 50, 640, 480   # bench.py's configs[1]
KCAM = (525.0, 525.0, 320.0, 240.0)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def pinned(ctype):
    """a ctypes array in pinned host memory, so that the device -> host copy of the records does not hold the submit"""
    import torch

    buf = torch.zeros(ctypes.sizeof(ctype), dtype=torch.uint8).pin_memory()
    arr = ctype.from_address(buf.data_ptr())
    arr._buf = buf
    return arr


def cameras(n, seed=1):
    """n distinct client cameras: K, the image size and a local transform (a yaw of the base, an offset, the optical rotation)"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        fx = rng.uniform(480, 640)
        K = (fx, fx * rng.uniform(0.98, 1.02), 320 + rng.uniform(-20, 20), 240 + rng.uniform(-20, 20))
        a = rng.uniform(-0.3, 0.3)
        L = np.eye(4)
        L[:3, :3] = [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]
        L[:3, 3] = rng.uniform(-0.5, 0.5, 3)
        O = np.eye(4)
        O[:3] = OPTICAL_ROTATION
        out.append(camera_model(K, (IMG_W, IMG_H), (L @ O)[:3]))
    return out


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
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
    h_img = [torch.from_numpy(np.ascontiguousarray(imgs[k * B:(k + 1) * B])).pin_memory() for k in range(args.pool)]
    h_dep = [torch.from_numpy(np.ascontiguousarray(deps[k * B:(k + 1) * B]).view(np.int16)).pin_memory() for k in range(args.pool)]
    dp = Engine.decide_params()
    clients = np.arange(B, dtype=np.int32)
    flags = np.zeros(B, np.int32)
    cams = cameras(B)
    op_c = [Engine.orb_params((c.fx, c.fy, c.cx, c.cy), n_features=F_FEATS) for c in cams]
    vp_c = [Engine.verify_params((c.fx, c.fy, c.cx, c.cy), image_size=(IMG_W, IMG_H)) for c in cams]
    out = [dict(nkp=torch.zeros(B, dtype=torch.int32).pin_memory().numpy(), words=torch.zeros(B * F_FEATS, dtype=torch.int32).pin_memory().numpy(),
                like=torch.zeros(B * ns, dtype=torch.float32).pin_memory().numpy(), dec=np.zeros(B, DECISION_DTYPE), res=pinned(VerifyResult * B))
           for _ in range(2)]

    def submit(k):
        o = out[k & 1]
        im, de = h_img[k % args.pool].numpy(), h_dep[k % args.pool].numpy().view(np.uint16)
        eng.process_frames_decide_submit(im, de, op, ns, ns + 1, vp, clients, flags, dp, None, o["nkp"], o["words"], o["like"], o["dec"], o["res"])

    def submit_one(k, f):
        o = out[(k * B + f) & 1]
        im, de = h_img[k % args.pool].numpy()[f:f + 1], h_dep[k % args.pool].numpy().view(np.uint16)[f:f + 1]
        eng.process_frames_decide_submit(im, de, op_c[f], ns, ns + 1, vp_c[f], clients[f:f + 1], flags[:1], dp, None, o["nkp"], o["words"],
                                         o["like"], o["dec"], o["res"])

    def run(kind, steps):
        eng.clients_set_cameras(clients, cams if kind == "distinct" else None)
        t = time.perf_counter()
        n = 0
        for k in range(steps):
            for f in (range(B) if kind == "per_client" else [None]):
                if f is None:
                    submit(k)
                else:
                    submit_one(k, f)
                if n >= 1:
                    eng.process_frames_wait()
                n += 1
        eng.process_frames_wait()
        return steps * B / (time.perf_counter() - t)

    arms = ("shared", "distinct", "per_client")
    for kind in arms:
        run(kind, args.warmup)
    rates = {kind: [] for kind in arms}
    for _ in range(args.rounds):
        for kind in arms:
            rates[kind].append(run(kind, args.steps))
    gpu = card()
    for kind in arms:
        r = rates[kind]
        print(f"{kind:10s} {min(r):9.0f} .. {max(r):9.0f} frames/s  ({gpu})")
    print(json.dumps({"gpu": gpu, "batch": B, "steps": args.steps, "rounds": args.rounds, "frames_per_s": rates}))


if __name__ == "__main__":
    main()
