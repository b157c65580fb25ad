"""Pin oracle/bayes_py.py to the reference's own BayesFilter.cpp, compiled by oracle/Makefile into oracle/_ref/libref_bayes.so against
the stand-ins of oracle/refstubs/ (cv::Mat, Memory::getNeighborsId from a loaded neighbour table, Parameters).

What is pinned: generatePrediction / addNeighborProb / normalize bit for bit (every float statement of the reference runs as
written), setPredictionLC's parsing, and the recursion of computePosterior / updatePosterior.  What is not: the cv::Mat product
(the stand-in accumulates in double, OpenCV's gemm order is not reproduced) and the graph walk of Memory (the tables are the test's).
The tests skip where the library could not be built (no copy of the reference to compile it from)."""
import zlib

import numpy as np
import pytest

from bayes_cases import GRAPHS, PATTERNS, likelihood, make_graph, n_levels, with_vp
from oracle import oracle_py as orc
from oracle.bayes_py import DEFAULT_PREDICTION_LC, BayesFilterOracle, parse_prediction_lc

pytestmark = pytest.mark.skipif(orc.ref_bayes_lib() is None, reason="oracle/_ref/libref_bayes.so is not built (no reference sources)")

SIZES = (1, 2, 3, 31, 33, 257, 600)


def dense_from_sparse(bf: BayesFilterOracle, ids, cols):
    """The matrix the sparse columns stand for, with the virtual-place row and column of generatePrediction / normalize."""
    col_ptr, rows, vals, u = cols
    n = len(ids)
    first = 1 if ids[0] < 0 else 0
    f = np.float32
    P = np.zeros((n, n), np.float32)
    for c in range(first, n):
        P[first:, c] = u[c]
        P[rows[col_ptr[c]:col_ptr[c + 1]], c] = vals[col_ptr[c]:col_ptr[c + 1]]
        if first:
            P[0, c] = f(bf.lc[0])
    if first:
        if bf.vpp > 0:
            P[0, 0] = bf.vpp if n > 1 else f(1)
            P[1:, 0] = f((1.0 - float(bf.vpp)) / (n - 1)) if n > 1 else 0
        else:
            P[:, 0] = f(1.0 / n) if n > 1 else f(1)
    return P


@pytest.mark.parametrize("graph", GRAPHS)
@pytest.mark.parametrize("pattern", list(PATTERNS))
def test_prediction_columns_equal_the_reference_bit_for_bit(pattern, graph):
    text = PATTERNS[pattern]
    rng = np.random.default_rng(zlib.crc32(f"{pattern}/{graph}".encode()))
    for k, (vpp, vp) in enumerate([(0.9, True), (0.0, True), (1.0, True), (0.9, False)]):
        n = SIZES[(k + len(pattern) + len(graph)) % len(SIZES)]
        places = list(range(1, n + 1 - vp)) if n - vp > 0 else []
        if not places:
            continue
        ids = with_vp(places, vp)
        tables, stm = make_graph(graph, places, n_levels(text), rng)
        ref = orc.RefBayesFilter(text, vpp)
        ref.set_graph(tables, stm)
        P_ref = ref.generate_prediction(ids)
        bf = BayesFilterOracle(text, vpp)
        P_dense = bf.prediction(ids, tables.__getitem__, stm)
        P_sparse = dense_from_sparse(bf, ids, bf.sparse_columns(ids, tables.__getitem__, stm))
        where = f"{pattern} {graph} n={len(ids)} vpp={vpp} vp={vp}"
        assert np.array_equal(P_ref.view(np.int32), P_dense.view(np.int32)), where
        assert np.array_equal(P_ref.view(np.int32), P_sparse.view(np.int32)), where


@pytest.mark.parametrize("pattern", ["default", "trunc5", "zerodiag", "largefill"])
@pytest.mark.parametrize("vp", [True, False])
def test_posterior_stream_equals_the_reference(pattern, vp):
    """Growth, removal and reactivation of places (a reactivated place starts again from 0), a reset, and an all-zero likelihood
    (the posterior stays unnormalised zeros, and so does the next one)."""
    text = PATTERNS[pattern]
    rng = np.random.default_rng(7 + vp)
    ref = orc.RefBayesFilter(text, 0.9)
    bf = BayesFilterOracle(text, 0.9)
    places = list(range(1, 41))
    removed = []
    for t in range(14):
        places.append(places[-1] + 1)
        if t % 4 == 3:                          # forget three places, bring back one forgotten earlier
            for v in rng.choice(places[3:-3], 3, replace=False):
                places.remove(int(v))
                removed.append(int(v))
            back = removed.pop(0)
            places = sorted(places + [back])
        if t == 9:
            ref.reset()
            bf.reset()
        ids = with_vp(places, vp)
        tables, stm = make_graph("loops" if t % 2 else "merged", places, n_levels(text), rng)
        like = likelihood(ids, t, rng)
        if t == 6:
            like[:] = 0
        ref.set_graph(tables, stm)
        p_ref = ref.compute_posterior(ids, like)
        p_orc = bf.compute_posterior_sparse(ids, like, tables.__getitem__, stm)
        assert np.allclose(p_orc, p_ref, rtol=1e-6, atol=1e-12), f"step {t}"
        if t in (6, 7):
            assert not p_ref.any()


def test_default_pattern_is_the_reference_default_rounded_through_float():
    ref = orc.RefBayesFilter(None)
    lc = ref.prediction_lc()
    assert np.array_equal(lc, np.array([np.float32(v) for v in DEFAULT_PREDICTION_LC], np.float64))
    assert np.array_equal(lc, parse_prediction_lc(PATTERNS["default"]))
    # _totalPredictionLCValues and _predictionEpsilon of the reference's values are the oracle's
    bf = BayesFilterOracle(PATTERNS["default"])
    total = np.float32(0)
    for v in lc:
        total = np.float32(float(total) + v)
    assert bf.total == total and bf.eps == np.float32(lc.min())
    assert float(bf.total) >= 1.0   # the default pattern needs no uniform fill
