"""NN-kernel tuning sweep on a real H100 : times the dictionary-NN kernel and
the fused quantise->score batch for the knob combinations given by env LCD_NN_* values."""
import itertools
import json
import os
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from rtabmap_b200 import Engine, synth  # noqa: E402

W = int(os.environ.get("SWEEP_W", 49152))
S = int(os.environ.get("SWEEP_S", 10000))
B = int(os.environ.get("SWEEP_B", 16))
F = 1000


def main():
    out = {}
    vocab = synth.make_binary_vocabulary(W)
    ids = np.arange(1, W + 1, dtype=np.int32)
    m = synth.make_map(ids, S, F)
    q, places = synth.make_query_frames(vocab, ids, m, B, F)
    dq = torch.from_numpy(q).cuda()
    dsig = torch.from_numpy(m.sig_ids).cuda()
    dwords = torch.zeros(B * F, dtype=torch.int32, device="cuda")
    dlike = torch.zeros(B * S, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    combos = list(itertools.product([1, 2, 4], [2, 4, 8], [0, 1, 2]))
    for m_, tq, var in combos:
        os.environ["LCD_NN_CTAS_PER_SM"] = str(m_)
        os.environ["LCD_NN_TQ"] = str(tq)
        os.environ["LCD_NN_VARIANT"] = str(var)
        eng = Engine(max_words=W, max_signatures=S + 1)
        eng.add_words(ids, vocab)
        eng.last_word_id = W
        eng.update()
        eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
        eng.profile_enable(True)
        for _ in range(3):
            eng.localize_batch_dev(dq.data_ptr(), B, F, dsig.data_ptr(), S, S + 1, dwords.data_ptr(), dlike.data_ptr())
        eng.synchronize()
        eng.profile_reset()
        t0 = time.perf_counter()
        iters = 10
        for _ in range(iters):
            eng.localize_batch_dev(dq.data_ptr(), B, F, dsig.data_ptr(), S, S + 1, dwords.data_ptr(), dlike.data_ptr())
        eng.synchronize()
        wall = (time.perf_counter() - t0) / iters
        res = {k: eng.profile_read(i) for i, k in enumerate(["nn", "resolve", "score"])}
        key = f"m{m_}_tq{tq}_v{var}"
        out[key] = {"wall_ms_per_batch": wall * 1e3, "frames_per_s": B / wall,
                    **{k + "_ms": v[0] / max(v[1], 1) for k, v in res.items()}}
        print(key, json.dumps(out[key]), flush=True)
        eng.close()
    Path("gpurun_out").mkdir(exist_ok=True)
    Path("gpurun_out/sweep_nn.json").write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
