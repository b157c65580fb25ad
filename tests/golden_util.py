"""Shared loaders of the golden data: tests/golden/tfidf_golden.json (made by tests/golden/make_tfidf_golden.py) and the stored
answers of the reference's own rtflann (tests/golden/ref_knn2.npz)."""
import hashlib
import json
import os
from pathlib import Path

import numpy as np

GOLD = json.loads((Path(__file__).parent / "golden" / "tfidf_golden.json").read_text())


def load_golden_into(d, remap):
    """Feed the golden inverted index into a dictionary-like object (oracle or engine)."""
    word_ids = sorted(int(w) for w in GOLD["words"])
    desc = np.zeros((len(word_ids), 32), np.uint8)
    desc[:, :4] = np.asarray(word_ids, dtype=np.uint32).view(np.uint8).reshape(-1, 4)
    d.add_words(word_ids, desc)
    d.update()
    rp = [0]
    sig, cnt = [], []
    for w in word_ids:
        for s, c in GOLD["words"][str(w)]:
            sig.append(remap(s))
            cnt.append(c)
        rp.append(len(sig))
    d.load_csr(word_ids, rp, sig, cnt)
    d.set_ni([remap(s) for s in GOLD["sig_ids"]], GOLD["ni"])


REF_KNN2 = Path(__file__).parent / "golden" / "ref_knn2.npz"
_ref_knn2 = None


def _digest(data: np.ndarray, queries: np.ndarray) -> str:
    h = hashlib.sha256()
    for a in (data, queries):
        a = np.ascontiguousarray(a)
        h.update(f"{a.dtype.str}{a.shape}".encode())
        h.update(memoryview(a).cast("B"))
    return h.hexdigest()[:24]


def ref_knn2(data: np.ndarray, queries: np.ndarray):
    """2-NN of `queries` over `data` as the reference's own rtflann LinearIndex answers it: (idx[nq,2] int64, dist[nq,2] float32).

    The answers for the inputs the tests use were computed by oracle/_ref/libref_flann.so (compiled from the reference's sources by
    oracle/Makefile) and are stored in tests/golden/ref_knn2.npz under a digest of the inputs, so the comparison needs no copy of the
    reference.  Where that library has been built, every stored answer is also checked against a live call; with
    LCD_RECORD_REF_KNN2=1 missing answers are computed by it and added to the file."""
    from oracle import oracle_py as orc

    global _ref_knn2
    if _ref_knn2 is None:
        _ref_knn2 = dict(np.load(REF_KNN2)) if REF_KNN2.exists() else {}
    key = _digest(data, queries)
    live = orc.ref_knn2(data, queries) if orc.ref_lib() is not None else None
    if key + "_idx" not in _ref_knn2:
        if live is None or not os.environ.get("LCD_RECORD_REF_KNN2"):
            raise KeyError(f"no stored rtflann answer for these inputs (digest {key}): the inputs differ from those the golden data was made from")
        _ref_knn2[key + "_idx"] = live[0].astype(np.int32)
        _ref_knn2[key + "_dist"] = live[1]
        np.savez_compressed(REF_KNN2, **_ref_knn2)
    idx = _ref_knn2[key + "_idx"].astype(np.int64)
    dist = _ref_knn2[key + "_dist"]
    if live is not None:
        assert np.array_equal(live[0], idx) and np.array_equal(live[1].view(np.uint32), dist.view(np.uint32)), "stored rtflann answer is stale"
    return idx, dist
