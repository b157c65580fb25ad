"""Record the reference's own rtflann answers for the 256-D cases of tests/test_float256.py into ref_knn2_f256.npz.

    python tests/golden/make_ref_knn2_f256.py      (needs oracle/_ref/libref_flann.so, built by oracle/Makefile from the reference)"""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path[:0] = [str(HERE.parent.parent), str(HERE.parent)]

from oracle import oracle_py as orc  # noqa: E402
from test_float256 import CASES, GOLDEN, knn2_case  # noqa: E402

if __name__ == "__main__":
    out = {}
    for rows, seed in CASES:
        idx, dist = orc.ref_knn2(*knn2_case(rows, seed))
        out[f"idx_{rows}"] = idx.astype(np.int32)
        out[f"dist_{rows}"] = dist
    np.savez_compressed(GOLDEN, **out)
    print(f"wrote {GOLDEN}")
