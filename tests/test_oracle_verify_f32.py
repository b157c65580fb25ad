"""Pin the oracle's float-descriptor pair matching (orcv_match_pair with desc_type = 1: RegistrationVis global matching through a
temporary VWDictionary, RegistrationVis.cpp:1482-1546) to an independent replay on the reference's own primitives: its compiled
rtflann for the index side (the FROM words once update() has indexed them) and cv::BFMatcher(NORM_L2SQR) for the words each side
creates.  This pins the temporary dictionary of float descriptors the way test_oracle_ref.py pins the quantiser loop.

The rtflann answers are stored in tests/golden/ref_knn2_match_f32.npz under a digest of the inputs, so the test needs no copy of the
reference; where oracle/Makefile has built oracle/_ref/libref_flann.so every stored answer is also checked against a live call, and
LCD_RECORD_REF_KNN2=1 adds missing answers."""
import os
from pathlib import Path

import numpy as np
import pytest

import test_oracle_ref
from golden_util import _digest
from oracle import oracle_py as orc
from test_oracle_ref import _replay_add_new_words

STORE = Path(__file__).parent / "golden" / "ref_knn2_match_f32.npz"
_stored = None


def _ref_knn2(data, queries):
    global _stored
    if _stored is None:
        _stored = dict(np.load(STORE)) if STORE.exists() else {}
    key = _digest(data, queries)
    live = orc.ref_knn2(data, queries) if orc.ref_lib() is not None else None
    if key + "_idx" not in _stored:
        if live is None or not os.environ.get("LCD_RECORD_REF_KNN2"):
            raise KeyError(f"no stored rtflann answer for these inputs (digest {key})")
        _stored[key + "_idx"] = live[0].astype(np.int32)
        _stored[key + "_dist"] = live[1]
        np.savez_compressed(STORE, **_stored)
    idx = _stored[key + "_idx"].astype(np.int64)
    dist = _stored[key + "_dist"]
    if live is not None:
        assert np.array_equal(live[0], idx) and np.array_equal(live[1].view(np.uint32), dist.view(np.uint32)), "stored rtflann answer is stale"
    return idx, dist


def _unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def make_pair(dim, seed):
    """FROM and TO sets with near-duplicates inside each side (intra-frame new-word dependencies, NNDR rejections), exact duplicates
    inside each side and across the sides (equal distances), and unrelated descriptors (new words)."""
    rng = np.random.default_rng(seed)
    base = _unit(rng.standard_normal((200, dim)))
    near_f = _unit(base[rng.integers(0, 200, 60)] + 0.05 * rng.standard_normal((60, dim)))
    F = np.concatenate([base, near_f, np.repeat(base[5:6], 4, 0)])
    rng.shuffle(F)
    fresh = _unit(rng.standard_normal((60, dim)))
    T = np.concatenate([_unit(F[rng.integers(0, len(F), 150)] + 0.02 * rng.standard_normal((150, dim))), fresh,
                        _unit(fresh[:30] + 0.05 * rng.standard_normal((30, dim))), F[10:30].copy()])
    T[1::9] = T[0]
    return F.astype(np.float32), T.astype(np.float32)


def replay_match_pair(F, T, nndr):
    """addNewWords(descriptorsFrom, 1) on an empty dictionary, update(), addNewWords(descriptorsTo, 2)."""
    from_ids, last = _replay_add_new_words(np.zeros(0, np.int32), np.zeros((0, F.shape[1]), np.float32), F, nndr, 0)
    new_ids, first = np.unique(from_ids, return_index=True)   # every FROM id is a new word: indexed in ascending id
    to_ids, _ = _replay_add_new_words(new_ids.astype(np.int32), F[first], T, nndr, last)
    return from_ids, to_ids, last


@pytest.mark.parametrize("dim", [64, 128])
@pytest.mark.parametrize("nndr", [0.8, 0.6])
def test_float_match_pair_against_reference_primitives(dim, nndr, monkeypatch):
    monkeypatch.setattr(test_oracle_ref, "ref_knn2", _ref_knn2)
    F, T = make_pair(dim, 7 * dim)
    want_f, want_t, n_words = replay_match_pair(F, T, nndr)
    got_f, got_t = orc.match_pair(F, T, nndr)
    assert np.array_equal(got_f, want_f)
    assert np.array_equal(got_t, want_t)
    # the scene reaches every branch: FROM descriptors matched to a word of their own frame, TO descriptors matched to FROM words,
    # TO descriptors creating words, and TO descriptors matched to a word created by an earlier TO descriptor
    assert len(np.unique(want_f)) < len(F)
    assert (want_t <= n_words).any() and (want_t > n_words).any()
    new_t = want_t[want_t > n_words]
    assert len(np.unique(new_t)) < len(new_t)
