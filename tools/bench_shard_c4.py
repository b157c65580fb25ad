"""Word-range sharding of the float configuration C4 (BASELINE configs[3]: 64-D float descriptors, 1 M words, 100 k signatures).

    python -m torch.distributed.run --nproc-per-node N tools/bench_shard_c4.py [--batch B --steps K --warmup W]

Every rank owns rows sharding.shard_rows(W, N, rank) of the dictionary and the posting lists of those words, brings its own B frames of
1000 descriptors (weak scaling, as the binary C2 job) and runs lcd_shard_localize_batch_dev over the library's NCCL communicator.  The
world and the frames are bench.py's c4_world / c4_queries (same seeds).  Printed as one JSON line per rank: frames/s, the rank's NN time
(lcd_profile), the exchange volumes per step computed from shapes, the card's name and power limit read in this run.  Rank 0 checks its
frames of the last step against lcd_localize_batch_dev on an unsharded engine on the same GPU (word ids and likelihood bit for bit).

With N = 1 the script also times lcd_shard_knn2_keys_dev of ONE shard of W/G rows over G x B frames of queries for G = 1, 2, 4, 8: the
search one rank runs in a G-rank job.  That is a single-GPU emulation of one rank's search, not a scaling measurement: it leaves out
the exchanges and the other ranks."""
import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from rtabmap_b200 import Engine, sharding, synth  # noqa: E402

DIM, FEATS, NNDR = 64, 1000, 0.8
PROF_NN = 0


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def c4_world(W, S):
    """bench.py c4_world: the same generator and seeds"""
    vocab = synth.make_float_vocabulary(W, DIM, 1)
    ids = np.arange(1, W + 1, dtype=np.int32)
    return vocab, ids, synth.make_map(ids, S, FEATS, seed=2)


def c4_queries(vocab, smap, n_frames, seed):
    """bench.py c4_queries: revisits of random signatures + N(0, 0.02) noise, a fifth replaced by unrelated descriptors"""
    rng = np.random.default_rng(seed)
    q = np.empty((n_frames, FEATS, DIM), np.float32)
    places = rng.integers(0, len(smap.sig_ids), n_frames)
    for f in range(n_frames):
        rows = smap.sig_words[places[f]].astype(np.int64) - 1
        d = vocab[rows] + rng.normal(0, 0.02, (FEATS, DIM)).astype(np.float32)
        idx = rng.permutation(FEATS)[:FEATS // 5]
        d[idx] = synth.make_float_vocabulary(len(idx), DIM, 1000 + seed * 100 + f)
        q[f] = d
    return q, places


def gpu_card(index):
    """name and power limit of the card, read now (nvidia-smi query only)"""
    out = {"name": torch.cuda.get_device_name(index)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", str(index)],
                           capture_output=True, text=True, timeout=30)
        pl, clk = [x.strip() for x in r.stdout.strip().split(",")[:2]]
        out.update(power_limit_w=float(pl), max_sm_clock_mhz=float(clk))
    except Exception as ex:  # noqa: BLE001 - the card's name is still worth printing
        out["power_limit_w"] = f"not read: {ex}"
    return out


def make_engine(vocab, ids, smap, r0, r1, batch_frames, with_index=True):
    e = Engine(device=torch.cuda.current_device(), desc_type=1, desc_dim=DIM, max_words=r1 - r0 + 4096,
               max_signatures=len(smap.sig_ids) + 2 if smap is not None else 16384, max_queries=FEATS, max_batch=batch_frames)
    for a in range(r0, r1, 1 << 18):
        b = min(r1, a + (1 << 18))
        e.add_words(ids[a:b], vocab[a:b])
    e.last_word_id = int(ids[-1])
    e.update()
    if r0:
        e.shard_set_row_offset(r0)
    if with_index:
        e.load_csr(*sharding.shard_csr(smap.word_ids, smap.row_ptr, smap.sig, smap.cnt, ids[r0:r1]) if (r0, r1) != (0, len(ids)) else
                   (smap.word_ids, smap.row_ptr, smap.sig, smap.cnt))
        e.set_ni(smap.sig_ids, smap.ni)
    return e


def time_events(fn, steps, stream):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    torch.cuda.synchronize()
    for k in range(steps):
        ev[k][0].record(stream)
        fn(k)
        ev[k][1].record(stream)
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in ev]


def emulate_one_rank_search(vocab, ids, B, steps, warmup):
    """lcd_shard_knn2_keys_dev of the first W/G rows over G x B frames: one rank's search in a G-rank job, on this one GPU"""
    W = len(ids)
    out = []
    for G in (1, 2, 4, 8):
        r0, r1 = sharding.shard_rows(W, G, 0)
        e = make_engine(vocab, ids, None, r0, r1, G * B, with_index=False)
        nq = G * B * FEATS
        rng = np.random.default_rng(40 + G)
        src = rng.integers(0, W, nq)     # queries near rows of the WHOLE dictionary, as the gathered frames of G ranks
        q = torch.from_numpy(vocab[src] + rng.normal(0, 0.02, (nq, DIM)).astype(np.float32)).cuda()
        keys = torch.zeros(nq * 2, dtype=torch.int64, device="cuda")
        stream = torch.cuda.ExternalStream(e.stream)
        for _ in range(warmup):
            e.shard_knn2_keys_dev(q.data_ptr(), nq, keys.data_ptr())
        torch.cuda.synchronize()
        assert e.nn_last_kernel == 1, "the fp16 filter did not run"
        e.profile_enable(True)
        e.profile_reset()
        ms = time_events(lambda k: e.shard_knn2_keys_dev(q.data_ptr(), nq, keys.data_ptr()), steps, stream)
        nn_ms, nn_n = e.profile_read(PROF_NN)
        e.profile_enable(False)
        fb = e.nn_f32_stats(nq)[0]
        out.append({"ranks_emulated": G, "shard_rows": r1 - r0, "queries": nq, "ms_per_call": float(np.median(ms)),
                    "nn_kernels_ms_per_call": nn_ms / max(steps, 1), "queries_per_s": nq / (np.median(ms) * 1e-3), "fallback_queries": int(fb)})
        log(f"emulated rank of {G}: {out[-1]}")
        del e, q, keys
        torch.cuda.synchronize()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--words", type=int, default=1_000_000)
    ap.add_argument("--signatures", type=int, default=100_000)
    ap.add_argument("--batch", type=int, default=32, help="frames per rank and step")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-emulation", action="store_true", help="skip the single-GPU emulation of one rank's search")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_shard_c4.py needs CUDA devices; there is no CPU fallback")
    rank, G = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    W, S, B = args.words, args.signatures, args.batch
    t0 = time.time()
    vocab, ids, smap = c4_world(W, S)
    q_all, places = c4_queries(vocab, smap, G * B, 3)
    q_mine = np.ascontiguousarray(q_all[rank * B:(rank + 1) * B])
    log(f"rank {rank}: world of {W} words / {S} signatures in {time.time() - t0:.0f} s")
    r0, r1 = sharding.shard_rows(W, G, rank)
    eng = make_engine(vocab, ids, smap, r0, r1, B)

    if G > 1:
        import torch.distributed as dist

        dist.init_process_group("gloo")
        uid = [Engine.shard_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        eng.shard_comm_init(uid[0], rank, G)
        dist.barrier()
    else:
        eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)

    stream = torch.cuda.ExternalStream(eng.stream)
    torch.cuda.set_stream(stream)
    d_q = torch.from_numpy(q_mine.reshape(-1, DIM)).cuda()
    d_sig = torch.from_numpy(smap.sig_ids).cuda()
    d_rowids = torch.from_numpy(ids).cuda()
    d_words = torch.zeros(B * FEATS, dtype=torch.int32, device="cuda")
    d_like = torch.zeros(B * S, dtype=torch.float32, device="cuda")

    def step(_k):
        eng.shard_localize_batch_dev(d_q.data_ptr(), B, FEATS, d_sig.data_ptr(), S, S + 1, d_rowids.data_ptr(), W, d_words.data_ptr(), d_like.data_ptr(),
                                     True, NNDR, True)

    for k in range(args.warmup):
        step(k)
    torch.cuda.synchronize()
    eng.profile_enable(True)
    eng.profile_reset()
    ms = time_events(step, args.steps, stream)
    nn_ms, nn_n = eng.profile_read(PROF_NN)
    eng.profile_enable(False)
    step_ms = float(np.median(ms))
    rows_all = G * B * FEATS
    line = {
        "config": "C4 float, word-range sharded: lcd_shard_localize_batch_dev", "words": W, "signatures": S, "ranks": G, "rank": rank,
        "shard_rows": r1 - r0, "frames_per_rank_and_step": B, "descriptors_per_frame": FEATS, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step_median": step_ms, "ms_per_step_min": float(np.min(ms)), "ms_per_step_max": float(np.max(ms)),
        "frames_per_s_this_rank": B / (step_ms * 1e-3), "frames_per_s_job": G * B / (step_ms * 1e-3),
        "nn_ms_per_step": nn_ms / max(args.steps, 1), "nn_kernels_per_step": nn_n / max(args.steps, 1),
        # exchange volumes of one step on one rank, from shapes (bytes this rank receives from the others / reduces)
        "exchange_bytes_per_step": {
            "all_gather_descriptors": (G - 1) * B * FEATS * DIM * 4,
            "all_to_all_keys": (G - 1) * B * FEATS * 16,
            "all_gather_word_ids": (G - 1) * B * FEATS * 4,
            "reduce_scatter_scores_input": G * B * S * 8,
        },
        "searched_queries_per_step_this_rank": rows_all,
        "gpu": gpu_card(local),
    }

    if rank == 0:
        # the last step's results of this rank's frames against the unsharded engine on the same GPU
        w_sh, l_sh = d_words.cpu().numpy(), d_like.cpu().numpy()
        ref = eng if G == 1 else make_engine(vocab, ids, smap, 0, W, B)
        w_ref = torch.zeros_like(d_words)
        l_ref = torch.zeros_like(d_like)
        ref_stream = torch.cuda.ExternalStream(ref.stream)
        with torch.cuda.stream(ref_stream):
            ref.localize_batch_dev(d_q.data_ptr(), B, FEATS, d_sig.data_ptr(), S, S + 1, w_ref.data_ptr(), l_ref.data_ptr(), True, NNDR, True)
        torch.cuda.synchronize()
        line["check_vs_unsharded"] = {"word_ids_equal": bool(np.array_equal(w_sh, w_ref.cpu().numpy())),
                                      "likelihood_bit_equal": bool(np.array_equal(l_sh.view(np.uint32), l_ref.cpu().numpy().view(np.uint32))),
                                      "new_words": int((w_sh > W).sum()),
                                      "top1_place_hit_rate": float(np.mean(smap.sig_ids[l_sh.reshape(B, S).argmax(1)] == smap.sig_ids[places[:B]]))}
        del ref
    eng.shard_comm_destroy()
    if G == 1 and not args.no_emulation:
        torch.cuda.set_stream(torch.cuda.default_stream())
        line["single_gpu_emulation_of_one_rank_search"] = {
            "note": "lcd_shard_knn2_keys_dev of one W/G-row shard over G x B frames on ONE GPU: one rank's search at G ranks; no exchange, "
                    "no other ranks, not a scaling measurement",
            "runs": emulate_one_rank_search(vocab, ids, B, args.steps, args.warmup)}
    print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(json.dumps(line) + "\n")
    if G > 1:
        import torch.distributed as dist

        dist.destroy_process_group()
    chk = line.get("check_vs_unsharded")
    return 0 if chk is None or (chk["word_ids_equal"] and chk["likelihood_bit_equal"]) else 1


if __name__ == "__main__":
    sys.exit(main())
