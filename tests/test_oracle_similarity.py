"""The CPU oracle of the similarity likelihood (Memory::computeLikelihood with Kp/TfIdfLikelihoodUsed=false) on hand cases:
EpipolarGeometry::findPairs, Signature::compareTo's bad-signature rule and totalWords, and the global-descriptor value."""
import math

import numpy as np
import pytest

from oracle import similarity_py as sim


def test_find_pairs_documented_example():
    # EpipolarGeometry.h:137-140: a=[1 2 3 4 6 6], b=[1 1 2 4 5 6 6] -> (1,1a) (2,2) (4,4) (6a,6a) (6b,6b), realPairsCount = 5
    a, b = [1, 2, 3, 4, 6, 6], [1, 1, 2, 4, 5, 6, 6]
    assert sim.find_pairs(a, b) == 5
    assert sim.find_pairs(b, a) == 5
    assert sim.engine_pairs(a, b) == 5


def test_duplicates_on_one_side_only():
    assert sim.find_pairs([7, 7, 7, 9], [7, 9, 9]) == 2
    assert sim.find_pairs([7, 9, 9], [7, 7, 7, 9]) == 2
    assert sim.find_pairs([3, 3, 3], [4, 4]) == 0


def test_negative_ids_never_pair_and_do_not_count():
    q, s = [-1, -2, 5, 6], [-1, -2, -3, 5]
    assert sim.find_pairs(s, q) == 1  # -1 and -2 are on both sides but are skipped (id >= 0 test)
    assert sim.valid_words(q) == 2 and sim.valid_words(s) == 1
    # totalWords = max(valid(q), valid(s)) = 2, not max(4, 4)
    assert sim.compare_to(q, s) == np.float32(0.5)
    assert sim.find_pairs(s, q, ignore_negative_ids=False) == 3


@pytest.mark.parametrize("q,s", [([-1, -5], [1, 2]), ([1, 2], [-1, 0]), ([], [1]), ([3], []), ([0], [0])])
def test_bad_signature_on_either_side_gives_zero(q, s):
    assert sim.is_bad_signature(q) or sim.is_bad_signature(s)
    assert sim.compare_to(q, s) == 0.0


def test_virtual_place_and_ids_not_in_memory_give_zero():
    words = {1: [1, 2, 3], 2: [2, 3, 4]}
    out = sim.compute_likelihood([1, 2, 3], [0, -1, 1, 2, 99], words)
    assert out.dtype == np.float32
    assert out.tolist() == [0.0, 0.0, 1.0, np.float32(2) / np.float32(3), 0.0]


def test_quotient_is_a_float_division():
    v = sim.compare_to([1, 2, 3, 4, 5, 6, 7], [1, 2, 3, 10, 11, 12, 13, 14, 15])
    assert v == np.float32(3) / np.float32(9) and v.dtype == np.float32


def test_mixed_global_descriptor_presence_falls_back_to_words():
    g = np.array([0.6, 0.8], np.float32)
    h = np.array([0.8, 0.6], np.float32)
    words = {1: [1, 2], 2: [1, 9], 3: [5]}
    gd = {1: h, 3: g}
    out = sim.compute_likelihood([1, 2], [1, 2, 3], words, q_gdesc=g, sig_gdesc=gd)
    assert out[0] == np.float32((sim.exact_dot(g, h) + 1.0) / 2.0)  # both carry one: the descriptor decides
    assert out[1] == np.float32(0.5)                                  # signature 2 has none: words
    assert out[2] == sim.gdesc_value(g, g) and out[2] > 0.99          # identical unit descriptors; the words would give 0
    out = sim.compute_likelihood([1, 2], [1, 3], words, q_gdesc=None, sig_gdesc=gd)
    assert out.tolist() == [1.0, 0.0]                                 # the query has none: words for every id


def test_non_normalised_descriptors_fail_the_reference_assert():
    g = np.array([-1.0, -1.0], np.float32)
    with pytest.raises(AssertionError, match="normalized"):
        sim.compare_to([1], [1], g, -g)


def test_id_zero_is_where_find_pairs_and_the_engine_differ():
    """findPairs tests id >= 0, so it pairs id 0 although id 0 is an invalid word (not counted in totalWords); the engine never
    pairs ids <= 0.  The quantiser never produces id 0 inside a signature, so this input does not arise from real frames."""
    q, s = [0, 5], [0, 5]
    assert sim.find_pairs(s, q) == 2 and sim.engine_pairs(s, q) == 1
    assert sim.compare_to(q, s) == np.float32(2.0)  # the reference: two pairs over totalWords = 1
    assert sim.compare_to(q, s, pairs=sim.engine_pairs) == np.float32(1.0)
    # with id 0 on one side only, or without id 0, the two rules agree
    for a, b in [([0, 5], [5, 6]), ([5, 5, -3], [5, -3]), ([1, 2, 3, 4, 6, 6], [1, 1, 2, 4, 5, 6, 6])]:
        assert sim.find_pairs(a, b) == sim.engine_pairs(a, b)


def test_dot_bound_is_the_recursive_summation_bound():
    rng = np.random.default_rng(1)
    for d in (1, 7, 128, 4096):
        q = rng.normal(size=d).astype(np.float32)
        s = rng.normal(size=d).astype(np.float32)
        exact = sim.exact_dot(q, s)
        assert sim.gamma(d) == pytest.approx(d * 2.0 ** -24 / (1 - d * 2.0 ** -24), rel=1e-15)
        # a sequential float32 sum of the products and a float64 one both stay inside the bound
        acc32 = np.float32(0)
        for a, b in zip(q, s):
            acc32 = np.float32(acc32 + np.float32(a * b))
        assert abs(float(acc32) - exact) <= sim.dot_bound(q, s)
        assert abs(float(np.dot(q.astype(np.float64), s.astype(np.float64))) - exact) <= sim.dot_bound(q, s)
        assert exact == math.fsum((q.astype(np.float64) * s.astype(np.float64)).tolist())
