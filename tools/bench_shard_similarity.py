"""The similarity likelihood (Kp/TfIdfLikelihoodUsed=false) in the word-range-sharded step: lcd_shard_localize_similarity_batch_dev.

    python -m torch.distributed.run --nproc-per-node N tools/bench_shard_similarity.py [--config c2|c2-gdesc|c4|all --batch B --steps K]

Configurations (every rank brings its own B frames, weak scaling as tools/bench_shard_c4.py):
  c2        binary 32-byte descriptors, 49 152 words, 10 000 places, 1000 features per frame, word pairs only;
  c2-gdesc  the same with a 4096-D global descriptor on every place and every frame (the dot products of the local frames);
  c4        bench_shard_c4.py's C4 world (64-D float descriptors, 1 M words, 100 000 places), word pairs only.
Each configuration prints one JSON line per rank: the median step time over --steps device-timed steps, the exchange volumes per step
computed from shapes, and the card's name and power limit read in this run.  Rank 0 checks the last step's frames against
lcd_localize_similarity_batch_dev on an unsharded engine on the same GPU (word ids and likelihood bit for bit).  A run on one GPU
(N = 1) times the step on a communicator of one rank: the exchanges are copies, so it is not a multi-GPU scaling figure."""
import argparse
import json
import os
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from bench_shard_c4 import c4_queries, c4_world, gpu_card, time_events  # noqa: E402
from rtabmap_b200 import Engine, sharding, synth  # noqa: E402

FEATS, NNDR, GD_DIM = 1000, 0.8, 4096


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def c2_world(W=49152, S=10000):
    vocab = synth.make_binary_vocabulary(W, 32, 1)
    ids = np.arange(1, W + 1, dtype=np.int32)
    return vocab, ids, synth.make_map(ids, S, FEATS, seed=2)


def make_engine(desc_type, vocab, ids, smap, r0, r1, B):
    e = Engine(device=torch.cuda.current_device(), desc_type=desc_type, desc_dim=vocab.shape[1], max_words=r1 - r0 + 4096,
               max_signatures=len(smap.sig_ids) + 2, max_queries=FEATS, max_batch=B)
    for a in range(r0, r1, 1 << 18):
        b = min(r1, a + (1 << 18))
        e.add_words(ids[a:b], vocab[a:b])
    e.last_word_id = int(ids[-1])
    e.update()
    if r0:
        e.shard_set_row_offset(r0)
    e.load_csr(*sharding.shard_csr(smap.word_ids, smap.row_ptr, smap.sig, smap.cnt, ids[r0:r1]) if (r0, r1) != (0, len(ids)) else
               (smap.word_ids, smap.row_ptr, smap.sig, smap.cnt))
    return e


def unit_rows(n, dim, seed):
    g = np.abs(np.random.default_rng(seed).normal(size=(n, dim))).astype(np.float32)
    return g / np.linalg.norm(g, axis=1, keepdims=True)


def run(config, rank, G, local, B, steps, warmup):
    t0 = time.time()
    if config == "c4":
        vocab, ids, smap = c4_world(1_000_000, 100_000)
        q_all, _ = c4_queries(vocab, smap, G * B, 3)
        desc_type = 1
    else:
        vocab, ids, smap = c2_world()
        q_all, _ = synth.make_query_frames(vocab, ids, smap, G * B, FEATS, seed=3)
        q_all = q_all.reshape(G * B, FEATS, 32)
        desc_type = 0
    W, S = len(ids), len(smap.sig_ids)
    q_mine = np.ascontiguousarray(q_all[rank * B:(rank + 1) * B])
    gd = config == "c2-gdesc"
    log(f"rank {rank} {config}: world of {W} words / {S} places in {time.time() - t0:.0f} s")
    r0, r1 = sharding.shard_rows(W, G, rank)
    eng = make_engine(desc_type, vocab, ids, smap, r0, r1, B)
    if G > 1:
        import torch.distributed as dist

        uid = [Engine.shard_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        eng.shard_comm_init(uid[0], rank, G)
        dist.barrier()
    else:
        eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)

    stream = torch.cuda.ExternalStream(eng.stream)
    torch.cuda.set_stream(stream)
    d_q = torch.from_numpy(q_mine.reshape(-1)).cuda()
    d_sig = torch.from_numpy(smap.sig_ids).cuda()
    d_rowids = torch.from_numpy(ids).cuda()
    d_words = torch.zeros(B * FEATS, dtype=torch.int32, device="cuda")
    d_like = torch.zeros(B * S, dtype=torch.float32, device="cuda")
    gd_kw, table, frames_gd = {}, None, None
    if gd:
        table = unit_rows(S, GD_DIM, 7)                                          # row k = place smap.sig_ids[k]
        frames_gd = unit_rows(G * B, GD_DIM, 8)[rank * B:(rank + 1) * B]
        d_tab = torch.from_numpy(table).cuda()
        d_row = torch.arange(S, dtype=torch.int32, device="cuda")
        d_fg = torch.from_numpy(np.ascontiguousarray(frames_gd)).cuda()
        gd_kw = dict(d_frame_gdesc=d_fg.data_ptr(), d_map_gdesc=d_tab.data_ptr(), d_map_gdesc_row=d_row.data_ptr(), n_map_rows=S, dim=GD_DIM)

    def step(_k):
        eng.shard_localize_similarity_batch_dev(d_q.data_ptr(), B, FEATS, d_sig.data_ptr(), S, d_rowids.data_ptr(), W, d_words.data_ptr(),
                                                d_like.data_ptr(), incremental=True, nndr=NNDR, cmp_new=True, **gd_kw)

    for k in range(warmup):
        step(k)
    torch.cuda.synchronize()
    ms = time_events(step, steps, stream)
    step_ms = float(np.median(ms))
    line = {
        "config": f"{config}: lcd_shard_localize_similarity_batch_dev", "words": W, "places": S, "ranks": G, "rank": rank, "shard_rows": r1 - r0,
        "frames_per_rank_and_step": B, "descriptors_per_frame": FEATS, "global_descriptor_dim": GD_DIM if gd else 0, "steps": steps,
        "warmup": warmup, "ms_per_step_median": step_ms, "ms_per_step_min": float(np.min(ms)), "ms_per_step_max": float(np.max(ms)),
        "frames_per_s_this_rank": B / (step_ms * 1e-3),
        # exchange volumes of one step on one rank, from shapes: bytes received from the other ranks, and the reduce-scatter's input
        "exchange_bytes_per_step": {
            "all_gather_descriptors": (G - 1) * B * FEATS * vocab.shape[1] * vocab.itemsize,
            "all_to_all_keys": (G - 1) * B * FEATS * (16 if desc_type == 1 else 8),
            "all_gather_word_ids": (G - 1) * B * FEATS * 4,
            "reduce_scatter_pairs_and_valid_input": G * (B + (2 if G >= 4 else 1)) * S * 4,
        },
        "gpu": gpu_card(local),
    }
    if rank == 0:
        w_sh, l_sh = d_words.cpu().numpy(), d_like.cpu().numpy()
        ref = eng if G == 1 else make_engine(desc_type, vocab, ids, smap, 0, W, B)
        if gd:
            ref.gdesc_add(smap.sig_ids, table)
        w_ref, l_ref = torch.zeros_like(d_words), torch.zeros_like(d_like)
        with torch.cuda.stream(torch.cuda.ExternalStream(ref.stream)):
            ref.localize_similarity_batch_dev(d_q.data_ptr(), B, FEATS, d_sig.data_ptr(), S, d_fg.data_ptr() if gd else 0, w_ref.data_ptr(),
                                              l_ref.data_ptr(), True, NNDR, True)
        torch.cuda.synchronize()
        line["check_vs_unsharded"] = {"word_ids_equal": bool(np.array_equal(w_sh, w_ref.cpu().numpy())),
                                      "likelihood_bit_equal": bool(np.array_equal(l_sh.view(np.uint32), l_ref.cpu().numpy().view(np.uint32))),
                                      "nonzero_likelihoods": int((l_sh > 0).sum())}
        if ref is not eng:
            del ref
    eng.shard_comm_destroy()
    torch.cuda.set_stream(torch.cuda.default_stream())
    del eng
    torch.cuda.synchronize()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="all", choices=["c2", "c2-gdesc", "c4", "all"])
    ap.add_argument("--batch", type=int, default=32, help="frames per rank and step")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_shard_similarity.py needs CUDA devices; there is no CPU fallback")
    rank, G = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    if G > 1:
        import torch.distributed as dist

        dist.init_process_group("gloo")
    ok = True
    for config in (["c2", "c2-gdesc", "c4"] if args.config == "all" else [args.config]):
        line = run(config, rank, G, local, args.batch, args.steps, args.warmup)
        print(json.dumps(line), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(line) + "\n")
        chk = line.get("check_vs_unsharded")
        ok = ok and (chk is None or (chk["word_ids_equal"] and chk["likelihood_bit_equal"]))
    if G > 1:
        import torch.distributed as dist

        dist.destroy_process_group()
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
