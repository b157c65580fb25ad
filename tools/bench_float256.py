"""Time the localisation step (quantise + TF-IDF score) of a C4-shaped world at 256-D (SuperPoint-sized rows) beside the 64-D C4 step.

    python tools/bench_float256.py [--batch 32 --steps 10 --warmup 3 --words 1000000 --signatures 100000] [--out result.json]

bench.py's C4 is fixed at 64-D.  This runs the same world twice, once with 64-D and once with 256-D unit rows from
synth.make_float_vocabulary: C4's word and signature counts, 1000 features per frame, frames built as bench.py builds them (rows of
the visited signature's words + N(0, 0.02) noise, a fifth replaced by unrelated descriptors).  For each width, one process and one
card, it reports:
  step_ms          lcd_localize_batch_dev on `batch` frames, CUDA events over `steps` back-to-back calls after `warmup` calls
                   (frames_per_s: bench.py's queries/s);
  cand_per_query   candidate rows the fp16 filter handed to the exact re-rank, per query (lcd_nn_f32_stats);
  fallback         queries redone by the exact scan in the last call (list overflow or values outside fp16);
  filter_ms        knn2_tensor_f32_kernel time per step (torch.profiler, a separate run of `steps` calls);
  filter_tflops    2 * nq * W * (D + 16) / filter_ms, and its share of the H100 SXM's 989 TFLOP/s dense fp16 figure.
One JSON line on stdout, with the card's name and power limit read in this run."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from rtabmap_b200 import Engine, synth  # noqa: E402

F = 1000
NNDR = 0.8
PEAK_FP16_TFLOPS = 989.0  # H100 SXM data sheet, dense, at a 700 W limit


def card():
    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=20)
        pl, clk = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        out.update(power_limit_w=float(pl), max_sm_clock_mhz=float(clk))
    except Exception as ex:
        out["power_limit_w"] = f"not read: {ex}"
    return out


def frames(vocab, smap, n_frames, seed):
    rng = np.random.default_rng(seed)
    dim = vocab.shape[1]
    q = np.empty((n_frames, F, dim), np.float32)
    for f in range(n_frames):
        rows = smap.sig_words[rng.integers(0, len(smap.sig_ids))].astype(np.int64) - 1
        d = vocab[rows] + rng.normal(0, 0.02, (F, dim)).astype(np.float32)
        idx = rng.permutation(F)[:F // 5]
        d[idx] = synth.make_float_vocabulary(len(idx), dim, 1000 + seed * 100 + f)
        q[f] = d
    return q


def run(dim, ids, smap, args):
    W, S, B = len(ids), len(smap.sig_ids), args.batch
    vocab = synth.make_float_vocabulary(W, dim, 1)
    eng = Engine(device=0, desc_type=1, desc_dim=dim, max_words=W + 4096, max_signatures=S + 2, max_queries=F, max_batch=B)
    eng.add_words(ids, vocab)
    eng.last_word_id = W
    eng.update()
    eng.load_csr(smap.word_ids, smap.row_ptr, smap.sig, smap.cnt)
    eng.set_ni(smap.sig_ids, smap.ni)
    pool = [torch.from_numpy(frames(vocab, smap, B, 3 + k).reshape(-1)).cuda() for k in range(2)]
    del vocab
    d_sig = torch.from_numpy(smap.sig_ids).cuda()
    d_words = torch.zeros(B * F, dtype=torch.int32, device="cuda")
    d_like = torch.zeros(B * S, dtype=torch.float32, device="cuda")
    k = [0]

    def step():  # on the engine's stream, where the events below are recorded
        eng.localize_batch_dev(pool[k[0] % 2].data_ptr(), B, F, d_sig.data_ptr(), S, S + 1, d_words.data_ptr(), d_like.data_ptr(), True, NNDR, True)
        k[0] += 1

    with torch.cuda.stream(torch.cuda.ExternalStream(eng.stream)):
        return measure(eng, step, dim, W, B, args)


def measure(eng, step, dim, W, B, args):

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.steps):
        step()
    t1.record()
    torch.cuda.synchronize()
    step_ms = t0.elapsed_time(t1) / args.steps
    nq = B * F
    n_fb, n_cand, _ = eng.nn_f32_stats(nq)
    filter_ran = eng.nn_last_kernel == 1
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    filt_us = sum(e.device_time_total for e in prof.key_averages() if "knn2_tensor_f32_kernel" in e.key)
    filter_ms = filt_us / 1000.0 / args.steps
    flops = 2.0 * nq * W * (dim + 16)
    out = {"dim": dim, "step_ms": round(step_ms, 3), "frames_per_s": round(B / (step_ms / 1000.0), 1),
           "cand_per_query": round(n_cand / nq, 2), "fallback": int(n_fb), "filter_ms": round(filter_ms, 3)}
    if filter_ms > 0:
        out["filter_tflops"] = round(flops / (filter_ms / 1000.0) / 1e12, 1)
        out["filter_share_of_989"] = round(flops / (filter_ms / 1000.0) / 1e12 / PEAK_FP16_TFLOPS, 3)
    out["filter_ran"] = filter_ran
    eng.close()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--words", type=int, default=1_000_000)
    ap.add_argument("--signatures", type=int, default=100_000)
    ap.add_argument("--out", type=str, default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_float256 needs a CUDA device")
    t = time.time()
    ids = np.arange(1, args.words + 1, dtype=np.int32)
    smap = synth.make_map(ids, args.signatures, F, seed=2)
    print(f"world: {args.words} words, {args.signatures} signatures in {time.time() - t:.0f} s", file=sys.stderr)
    res = {"tool": "bench_float256", "words": args.words, "signatures": args.signatures, "features_per_frame": F, "frames_per_step": args.batch,
           "steps": args.steps, "warmup": args.warmup, **card()}
    res["d256"] = run(256, ids, smap, args)
    res["d64"] = run(64, ids, smap, args)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
