"""Time the verification kernels on a H100.

    python tools/time_verify.py [pairs [outlier_fraction]]     # 128 pairs at 0.3 outliers run 36-95 RANSAC iterations; at 0.1, under 16

With LCD_PNP_CLOCKS=1 it also prints thread 0's clock64 phases of pnp_ransac_kernel: RANSAC's first wave of hypotheses (kPnpWave,
verify.cuh), the second wave (kPnpWaveMax), which only runs when the run goes past the first, and any later waves."""
import json
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
from rtabmap_b200 import Engine  # noqa: E402
from rtabmap_b200.capi import LcdError  # noqa: E402
from test_gpu_verify import make_pair, K4  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
OUTLIERS = float(sys.argv[2]) if len(sys.argv) > 2 else 0.3
rng = np.random.default_rng(0)
cap = 1000
F = np.zeros((B, cap, 32), np.uint8); T = np.zeros((B, cap, 32), np.uint8)
X = np.zeros((B, cap, 3), np.float32); U = np.zeros((B, cap, 2), np.float32)
for i in range(B):
    F[i], X[i], T[i], U[i] = make_pair(rng, cap, outlier_frac=OUTLIERS)
eng = Engine()
eng.profile_enable(True)
for _ in range(2):
    out = eng.verify_batch(F, X, T, U, K4)
eng.profile_reset()
t0 = time.perf_counter()
n = 5
for _ in range(n):
    out = eng.verify_batch(F, X, T, U, K4)
dt = (time.perf_counter() - t0) / n
m = eng.profile_read(3); p = eng.profile_read(4)
print(json.dumps({"pairs": B, "outlier_fraction": OUTLIERS, "wall_ms": dt * 1e3, "pairs_per_s": B / dt, "match_ms": m[0] / m[1], "pnp_ms": p[0] / p[1],
                  "ok": sum(o["ok"] for o in out), "inliers": [len(o["inliers"]) for o in out[:4]], "iters": [o["iterations_run"] for o in out[:8]]}))
clk = eng.debug_orb_buffer(7, B * 16 * 8, np.int64).reshape(B, 16)
d = np.diff(clk[:, :5], axis=1).astype(np.float64)
print(json.dumps({"pnp_phase_kcycles_mean": {k: round(float(v) / 1e3, 1) for k, v in zip(("sample", "waves1_2", "later_waves", "refine"), d.mean(0))},
                  "pnp_phase_kcycles_max": {k: round(float(v) / 1e3, 1) for k, v in zip(("sample", "waves1_2", "later_waves", "refine"), d.max(0))}}))
w = np.stack([clk[:, 5] - clk[:, 1], clk[:, 2] - clk[:, 5]], 1).astype(np.float64)
iters = np.array([o["iterations_run"] for o in out])
past = iters > 16
print(json.dumps({"wave1_kcycles_mean": round(float(w[:, 0].mean()) / 1e3, 1), "wave1_kcycles_max": round(float(w[:, 0].max()) / 1e3, 1),
                  "pairs_past_wave1": int(past.sum()),
                  "wave2_kcycles_mean": round(float(w[past, 1].mean()) / 1e3, 1) if past.any() else None,
                  "wave2_kcycles_max": round(float(w[past, 1].max()) / 1e3, 1) if past.any() else None}))
e = np.diff(clk[:, 8:14], axis=1).astype(np.float64)
print(json.dumps({"epnp_thread0_kcycles_mean": {k: round(float(v) / 1e3, 1) for k, v in zip(("ctrl+MtM", "eigen12", "betas+GN+Rt", "m2v", "count"), e.mean(0))}}))
g = eng.debug_orb_buffer(8, 64, np.int64)
print(json.dumps({"last_writer_kcycles": {"tred2": g[0] / 1e3, "gn": [g[2] / 1e3, g[3] / 1e3, g[4] / 1e3], "Rt": [g[5] / 1e3, g[6] / 1e3, g[7] / 1e3]}}))
try:
    g = eng.debug_orb_buffer(9, 64, np.int64)  # the matching kernel's clocks exist only in a build with LCD_DEBUG_PHASES
except LcdError:
    sys.exit(0)
print(json.dumps({"match_block0_kcycles": dict(zip(("from_resolve", "dict_build", "to_knn", "to_resolve", "correspondences"), (np.diff(g[:6]) / 1e3).round(1).tolist()))}))
