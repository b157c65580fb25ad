"""Time the similarity likelihood (lcd_localize_similarity_batch_dev) against the TF-IDF one (lcd_localize_batch_dev) on a C2-shaped map.

    python tools/bench_similarity.py [--batch 128 --steps 20 --warmup 5 --dim 4096]

The map has C2's sizes (49 152 binary words, 10 000 signatures of 1000 words, synth.make_map) and B frames of 1000 descriptors
revisiting it (synth.make_query_frames).  Three calls are timed with CUDA events after warm-up, each over `steps` back-to-back calls:
  tfidf       lcd_localize_batch_dev: quantise + TF-IDF likelihood;
  sim_words   lcd_localize_similarity_batch_dev with no global descriptors: quantise + word pairs;
  sim_gdesc   the same with a unit `dim`-D global descriptor on every signature and every frame (the dense B x 10 000 x dim product).
sim_gdesc_ms - sim_words_ms is what the global descriptors add to the call (the dot-product kernel); gdesc_gflop is the product's
work computed from shapes.  One JSON line on stdout, with the card's name and power limit read in this run."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dim", type=int, default=4096)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_similarity needs a CUDA device")
    B, D = args.batch, args.dim
    vocab = synth.make_binary_vocabulary(W, 32, 1)
    ids = np.arange(1, W + 1, dtype=np.int32)
    m = synth.make_map(ids, S, F, seed=2)
    q, places = synth.make_query_frames(vocab, ids, m, B, F, seed=3)
    eng = Engine(max_words=W, max_signatures=S + 2, max_queries=F, max_batch=B)
    eng.add_words(ids, vocab)
    eng.last_word_id = W
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    eng.set_ni(m.sig_ids, m.ni)
    rng = np.random.default_rng(7)
    G = rng.normal(size=(S, D)).astype(np.float32)
    G /= np.linalg.norm(G, axis=1, keepdims=True)
    Q = G[places - 1] + 0.3 * rng.normal(size=(B, D)).astype(np.float32) / np.sqrt(D)
    Q = (Q / np.linalg.norm(Q, axis=1, keepdims=True)).astype(np.float32)

    st = eng.stream
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_s = torch.from_numpy(m.sig_ids).cuda()
    d_g = torch.from_numpy(Q.reshape(-1)).cuda()
    d_w = torch.zeros(B * F, dtype=torch.int32, device="cuda")
    d_l = torch.zeros(B * S, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()

    def tfidf():
        eng.localize_batch_dev(d_q.data_ptr(), B, F, d_s.data_ptr(), S, S + 1, d_w.data_ptr(), d_l.data_ptr(), stream=st)

    def sim(g=0):
        eng.localize_similarity_batch_dev(d_q.data_ptr(), B, F, d_s.data_ptr(), S, g, d_w.data_ptr(), d_l.data_ptr(), stream=st)

    # time on the engine's stream: torch events record on the current stream, so make it the engine's
    ext = torch.cuda.ExternalStream(st)
    res = {"batch": B, "frames_desc": F, "words": W, "signatures": S, "gdesc_dim": D, "steps": args.steps, "warmup": args.warmup}
    with torch.cuda.stream(ext):
        res["tfidf_ms"] = time_ms(tfidf, args.steps, args.warmup)
        res["sim_words_ms"] = time_ms(sim, args.steps, args.warmup)
        l_words = d_l.cpu().numpy().reshape(B, S).copy()
        eng.gdesc_add(m.sig_ids, G)
        res["sim_gdesc_ms"] = time_ms(lambda: sim(d_g.data_ptr()), args.steps, args.warmup)
        l_g = d_l.cpu().numpy().reshape(B, S)
    res["gdesc_added_ms"] = res["sim_gdesc_ms"] - res["sim_words_ms"]
    res["gdesc_gflop"] = 2.0 * B * S * D / 1e9
    res["gdesc_bytes_rows_mb"] = S * D * 4 / 1e6
    res["sim_words_top1_is_place"] = float(np.mean(m.sig_ids[np.argmax(l_words, 1)] == places))
    res["sim_gdesc_top1_is_place"] = float(np.mean(m.sig_ids[np.argmax(l_g, 1)] == places))
    res.update(card())
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
