"""RANSAC iterations per verified pair in bench.py's workloads: how far each PnP RANSAC run gets before the reference's adaptive
iteration count stops it.  `pnp_ransac_kernel` solves the hypotheses of a chunk in waves (verify.cuh), and a step waits for its
slowest pair, so what matters is the maximum over the 128 pairs of each step, not the mean.

    python tools/pnp_iterations.py            # one JSON line per frame pool: the headline's three, then the mixed workload's
"""
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from rtabmap_b200 import Engine, synth  # noqa: E402


def main():
    import torch

    B, n_pool = 128, 3
    eng = Engine(desc_dim=bench.DESC_BYTES, max_words=bench.W_WORDS + 65536, max_signatures=bench.S_SIGS + 128, max_queries=bench.F_FEATS,
                 max_batch=B)
    op = Engine.orb_params(bench.KCAM, n_features=bench.F_FEATS)
    vp = Engine.verify_params(bench.KCAM, image_size=(bench.IMG_W, bench.IMG_H))
    world = synth.make_place_world(lambda img, dep: eng.orb_detect_describe(img[None], dep[None], op, cap=bench.F_FEATS)[0], bench.N_PLACES,
                                   bench.W_WORDS, bench.S_SIGS, bench.F_FEATS, bench.IMG_H, bench.IMG_W)
    sm = world.smap
    eng.add_words(world.word_ids, world.vocab)
    eng.last_word_id = bench.W_WORDS
    eng.update()
    eng.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    eng.set_ni(sm.sig_ids, sm.ni)
    for s0 in range(0, bench.S_SIGS, 1000):
        eng.sig_add_batch(sm.sig_ids[s0:s0 + 1000], world.store.desc[s0:s0 + 1000], world.store.xyz[s0:s0 + 1000], sm.ni[s0:s0 + 1000])
    torch.cuda.set_stream(torch.cuda.ExternalStream(eng.stream))
    d_sig = torch.from_numpy(sm.sig_ids).cuda()
    d_w = torch.zeros(B * bench.F_FEATS, dtype=torch.int32, device="cuda")
    d_l = torch.zeros(B * bench.S_SIGS, dtype=torch.float32, device="cuda")

    def run(name, imgs, deps):
        d_i = torch.from_numpy(np.ascontiguousarray(imgs)).cuda()
        d_d = torch.from_numpy(np.ascontiguousarray(deps).view(np.int16)).cuda()
        eng.process_frames_dev(d_i.data_ptr(), B, bench.IMG_W, bench.IMG_H, 3, d_d.data_ptr(), 1, op, d_sig.data_ptr(), bench.S_SIGS,
                               bench.S_SIGS + 1, vp, d_w.data_ptr(), d_l.data_ptr(), True, bench.NNDR, True)
        torch.cuda.synchronize()
        _, res = eng.process_fetch(B)
        it = np.array([r["iterations_run"] for r in res])
        print(json.dumps({"pool": name, "max": int(it.max()), "p50": float(np.percentile(it, 50)), "p95": float(np.percentile(it, 95)),
                          "over_16": int((it > 16).sum()), "over_32": int((it > 32).sum()), "over_128": int((it > 128).sum()),
                          "counts": {int(k): int(v) for k, v in zip(*np.unique(it, return_counts=True))}}), flush=True)

    imgs, deps, _ = synth.make_view_frames(world, B * n_pool, seed=3, mode="revisit")
    for k in range(n_pool):
        run(f"headline_{k}", imgs[k * B:(k + 1) * B], deps[k * B:(k + 1) * B])
    imgs, deps, _ = synth.make_view_frames(world, B, seed=77, mode="mixed")
    run("mixed", imgs, deps)


if __name__ == "__main__":
    main()
