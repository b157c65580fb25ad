"""CPU restatement of the similarity branch of Memory::computeLikelihood (Kp/TfIdfLikelihoodUsed=false), test infrastructure only.

Memory::computeLikelihood (corelib/src/Memory.cpp:2179-2214) returns, for every id of the list in list order, 0 for ids <= 0 (the
virtual place) and Signature::compareTo (Signature.cpp:250-288) otherwise.  compareTo uses the global descriptors when both
signatures carry one of type 1, and the word pairs of EpipolarGeometry::findPairs (EpipolarGeometry.h:119-151) otherwise.  A
signature is given here as its word ids (a multiset: the keys of Signature::getWords()) and an optional global descriptor.

The global-descriptor value of the reference depends on how OpenCV's dotProd_32f is dispatched on the CPU, so the oracle gives the
exact dot product (math.fsum of the exact float64 products) and the rigorous bound of any fp32 recursive summation around it.
"""
from __future__ import annotations

import math
from collections import Counter

import numpy as np

U32 = 2.0 ** -24  # unit round-off of float32


def unique_keys(words) -> list[int]:
    """uUniqueKeys of a std::multimap: the distinct ids in ascending order."""
    return sorted(set(int(w) for w in words))


def find_pairs(words_a, words_b, ignore_negative_ids: bool = True) -> int:
    """EpipolarGeometry::findPairs(wordsA, wordsB, pairs, ignoreNegativeIds) -> realPairsCount, restated literally: for every
    unique id of A (id >= 0 when ignoring negatives) walk the equal ranges of both multimaps together, one pair per step."""
    ca, cb = Counter(int(w) for w in words_a), Counter(int(w) for w in words_b)
    count = 0
    for i in unique_keys(words_a):
        if not ignore_negative_ids or i >= 0:
            count += min(ca[i], cb.get(i, 0))
    return count


def engine_pairs(words_a, words_b) -> int:
    """The engine's rule: ids <= 0 never pair (its inverted index holds positive ids only).  Differs from find_pairs only when
    both sides contain id 0, which the quantiser never produces."""
    ca, cb = Counter(int(w) for w in words_a if w > 0), Counter(int(w) for w in words_b if w > 0)
    return sum(min(c, cb.get(i, 0)) for i, c in ca.items())


def invalid_words(words) -> int:
    """Signature::_invalidWordsCount: the ids <= 0 (Signature.cpp:320-330)."""
    return int(sum(1 for w in words if w <= 0))


def valid_words(words) -> int:
    return len(words) - invalid_words(words)


def is_bad_signature(words) -> bool:
    """Signature::isBadSignature (Signature.cpp:341-344)."""
    return valid_words(words) <= 0


def exact_dot(q, s) -> float:
    """The dot product of two float32 vectors, correctly rounded to float64 (each product is exact in float64)."""
    q = np.asarray(q, np.float32).astype(np.float64)
    s = np.asarray(s, np.float32).astype(np.float64)
    return math.fsum((q * s).tolist())


def gamma(d: int) -> float:
    """gamma_D = D u / (1 - D u): the relative bound of a D-term fp32 recursive (or FMA-chain) summation."""
    return d * U32 / (1.0 - d * U32)


def dot_bound(q, s) -> float:
    """|fp32 dot - exact dot| <= gamma_D * sum |q_i s_i| for any summation order of D fp32 fused multiply-adds."""
    q = np.asarray(q, np.float32).astype(np.float64)
    s = np.asarray(s, np.float32).astype(np.float64)
    return gamma(len(q)) * math.fsum(np.abs(q * s).tolist())


def gdesc_value(q, s) -> np.float32:
    """compareTo's global-descriptor value on the exact dot product: float((dot + 1.0f) / 2.0f)."""
    return np.float32((exact_dot(q, s) + 1.0) / 2.0)


def gdesc_value_tolerance(q, s, value) -> float:
    """How far a likelihood computed from an fp32 dot within dot_bound may lie from (exact + 1) / 2: half the dot bound plus the
    rounding of the final cast to float (at most half an ulp; one ulp of the value is allowed so a binade edge is covered)."""
    return dot_bound(q, s) / 2.0 + float(np.spacing(np.float32(abs(value))))


def compare_to(q_words, s_words, q_gdesc=None, s_gdesc=None, pairs=find_pairs) -> np.float32:
    """Signature::compareTo(s) called on the query q (Signature.cpp:250-288), one global descriptor per signature."""
    if q_gdesc is not None and s_gdesc is not None:
        v = gdesc_value(q_gdesc, s_gdesc)
        assert v >= 0, "Global descriptors should be normalized!"
        return v
    if is_bad_signature(s_words) or is_bad_signature(q_words):
        return np.float32(0.0)
    total = max(valid_words(q_words), valid_words(s_words))
    assert total > 0
    return np.float32(pairs(s_words, q_words)) / np.float32(total)


def compute_likelihood(q_words, ids, sig_words, q_gdesc=None, sig_gdesc=None, pairs=find_pairs) -> np.ndarray:
    """Memory::computeLikelihood with Kp/TfIdfLikelihoodUsed=false: sig_words / sig_gdesc map an id to its word ids / its global
    descriptor (absent = none).  The reference aborts on an id that is not in memory (UFATAL); here such an id is an empty
    signature, i.e. a bad one, which gives 0 as on the engine."""
    sig_gdesc = sig_gdesc or {}
    out = np.zeros(len(ids), np.float32)
    for k, i in enumerate(ids):
        i = int(i)
        if i > 0:
            out[k] = compare_to(q_words, sig_words.get(i, ()), q_gdesc, sig_gdesc.get(i), pairs)
    return out
