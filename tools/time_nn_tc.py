"""Time the binary dictionary 2-NN (knn2_tensor_kernel) at the shape bench.py times: its world of 49 152 words, and the ORB descriptors
of 128 of its 640x480 RGB-D frames as queries (~1000 per frame).  The kernel is timed with the engine's CUDA events around every launch
(lcd_profile_*, class "nn") over --launches calls of lcd_shard_knn2_keys_dev after --warmup calls.  Prints one JSON line: ms per launch,
cycles per SM and 256-query tile at the card's max SM clock, and the card's name, power limit and clocks, read in the same run.

    python tools/time_nn_tc.py [--launches 100] [--warmup 10] [--popc]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402  (the world's constants)

TILE_Q, TILE_W = 256, 256   # nn_tensor.cuh: kTcBM, kTcBN


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True)
    name, power, max_sm, sm = [x.strip() for x in q.stdout.strip().split(",")]
    return {"gpu": torch.cuda.get_device_name(0) or name, "power_limit_w": float(power), "max_sm_mhz": float(max_sm), "sm_mhz_now": float(sm),
            "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--popc", action="store_true", help="also time the POPC kernel (knn2_hamming_kernel) on the same queries")
    args = ap.parse_args()
    assert args.launches >= 50, "time at least 50 launches"

    import torch

    from rtabmap_b200 import Engine, synth

    if not torch.cuda.is_available():
        raise SystemExit("time_nn_tc.py needs a CUDA device")
    eng = Engine(desc_dim=bench.DESC_BYTES, max_words=bench.W_WORDS, max_queries=bench.F_FEATS, max_batch=args.frames)
    op = Engine.orb_params(bench.KCAM, n_features=bench.F_FEATS)

    def orb(img, dep):
        return eng.orb_detect_describe(img[None], dep[None], op, cap=bench.F_FEATS)[0]

    world = synth.make_place_world(orb, bench.N_PLACES, bench.W_WORDS, bench.S_SIGS, bench.F_FEATS, bench.IMG_H, bench.IMG_W)
    imgs, deps, _ = synth.make_view_frames(world, args.frames, seed=3)
    eng.add_words(world.word_ids, world.vocab)
    eng.last_word_id = bench.W_WORDS
    eng.update()
    q = np.concatenate([f[1] for f in eng.orb_detect_describe(imgs, deps, op, cap=bench.F_FEATS)])
    nq, n_rows = len(q), len(world.vocab)
    d_q = torch.from_numpy(np.ascontiguousarray(q).reshape(-1)).cuda()
    d_k = torch.zeros(nq * 2, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    info = card()
    out = {"frames": args.frames, "queries": nq, "words": n_rows, "launches": args.launches}

    def timed(kernel):
        eng.nn_select(kernel)
        for _ in range(args.warmup):
            eng.shard_knn2_keys_dev(d_q.data_ptr(), nq, d_k.data_ptr())
        eng.synchronize()
        eng.profile_enable(True)
        eng.profile_reset()
        for _ in range(args.launches):
            eng.shard_knn2_keys_dev(d_q.data_ptr(), nq, d_k.data_ptr())
        eng.synchronize()
        ms, n = eng.profile_read(0)
        eng.profile_enable(False)
        assert eng.nn_last_kernel == kernel and n == args.launches, (eng.nn_last_kernel, n)
        return ms / n, d_k.cpu().clone()

    ms, keys = timed(1)
    tiles_per_sm = -(-nq // TILE_Q) * -(-n_rows // TILE_W) / info["sms"]
    out.update(knn2_tensor_ms=round(ms, 4), cycles_per_sm_and_tile=round(ms * 1e-3 * info["max_sm_mhz"] * 1e6 / tiles_per_sm, 1),
               tiles_per_sm=round(tiles_per_sm, 1))
    if args.popc:
        p_ms, p_keys = timed(0)
        out.update(knn2_hamming_ms=round(p_ms, 4), keys_equal=bool(torch.equal(keys, p_keys)))
    info["sm_mhz_after"] = card()["sm_mhz_now"]
    print(json.dumps({**out, **info}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
